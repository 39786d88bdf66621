"""Digest of every kernel's machine code in the built objects (tools, not product): one line per kernel,
`object kernel sha256 resources`, sorted.  Two builds whose outputs are equal run the same instructions with the same
registers, shared, local and constant memory -- the way to show, without a GPU, that a change to host code or to a shared
device helper left every kernel as it was.

    python tools/sass_digest.py [build/obj] > after.txt      # then diff against the output at the other commit

Kernel names are demangled, and the per-translation-unit hash nvcc puts into internal-linkage names is replaced by a fixed
token, so moving code inside a file does not show up as a renamed kernel.
"""
import hashlib
import os
import re
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_TU_HASH = re.compile(r"(_INTERNAL_|_GLOBAL__N__|_cu_)[0-9a-f]{8}")


def _tool(name):
    path = shutil.which(name) or os.path.join("/usr/local/cuda/bin", name)
    if not os.path.isfile(path):
        raise RuntimeError("%s not found" % name)
    return path


def _run(args):
    return subprocess.run(args, check=True, capture_output=True, text=True).stdout


def _demangle(names):
    """mangled -> demangled, with the translation-unit hash (where the demangled name still shows it) replaced"""
    out = _run([_tool("cu++filt")] + names).splitlines() if names else []
    return dict(zip(names, (_TU_HASH.sub(r"\g<1>TU", n) for n in out)))


def _sass(obj):
    """mangled kernel name -> sha256 of its instruction text"""
    text = {}
    cur = None
    for line in _run([_tool("cuobjdump"), "-sass", obj]).splitlines():
        s = line.strip()
        if s.startswith("Function :"):
            cur = s.split(":", 1)[1].strip()
            text[cur] = []
        elif cur is not None and s.startswith("/*"):
            text[cur].append(" ".join(s.split()))       # address, instruction and its encoding (with the scheduling word)
    return {k: hashlib.sha256(_TU_HASH.sub(r"\g<1>TU", "\n".join(v)).encode()).hexdigest() for k, v in text.items()}


def _resources(obj):
    """mangled kernel name -> 'REG:.. STACK:.. SHARED:.. LOCAL:.. CONSTANT[0]:..' line"""
    res = {}
    cur = None
    for line in _run([_tool("cuobjdump"), "--dump-resource-usage", obj]).splitlines():
        s = line.strip()
        if s.startswith("Function "):
            cur = s[len("Function "):].rstrip(":")
        elif cur is not None and s.startswith("REG:"):
            res[cur] = " ".join(f for f in s.split() if not f.startswith(("TEXTURE", "SURFACE", "SAMPLER")))
            cur = None
    return res


def digest(obj_dir):
    lines = []
    for f in sorted(os.listdir(obj_dir)):
        if not f.endswith(".o"):
            continue
        obj = os.path.join(obj_dir, f)
        sass, res = _sass(obj), _resources(obj)
        if set(sass) != set(res):
            raise RuntimeError("%s: SASS and resource listings name different functions" % f)
        names = _demangle(sorted(sass))
        for k in sass:
            lines.append("%s %s %s %s" % (f, names[k].replace(" ", ""), sass[k], res[k]))
    return sorted(lines)


if __name__ == "__main__":
    print("\n".join(digest(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "build", "obj"))))
