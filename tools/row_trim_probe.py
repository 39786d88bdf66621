"""Does a 2-D tensor load of only the history columns of each observation row save DRAM time over one 1-D bulk copy of the
whole span?  Builds tools/row_trim_probe.cu (a copy-only model of step_pipe_kernel, DESIGN.md 4.1) for sm_90a in a temporary
directory, checks that every variant writes the same bytes, then times, variants alternating, µs per launch of 65 536 rows
(8 rotating buffer sets, as bench.py) and of 1 048 576 rows.  Prints the card (name, power limit, max SM clock) first and a
summary (best run per variant, saving against the 1-D copy) last.

    python tools/row_trim_probe.py [--runs 3] [--reps 2000]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))


def card():
    try:
        q = "name,power.limit,clocks.max.sm"
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return dict(zip(q.split(","), [c.strip() for c in out.strip().split(",")]))
    except Exception as ex:  # noqa: BLE001
        return {"error": repr(ex)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--reps", type=int, default=2000)
    a = ap.parse_args()
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "row_trim_probe")
        subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe, os.path.join(HERE, "row_trim_probe.cu")], check=True)
        print(json.dumps({"card": card()}), flush=True)
        p = subprocess.run([exe, str(a.runs), str(a.reps)], capture_output=True, text=True)
    sys.stdout.write(p.stdout)
    if p.returncode != 0:
        sys.stderr.write(p.stderr)
        raise SystemExit(p.returncode)
    best = {}
    for line in p.stdout.splitlines():
        r = json.loads(line)
        if "us_per_launch" in r:
            k = (r["N"], r["variant"])
            best[k] = min(best.get(k, float("inf")), r["us_per_launch"])
    summary = {}
    for (n, v), us in best.items():
        base = best[(n, "bulk")]
        summary.setdefault(str(n), {})[v] = {"best_us": us, "saving_pct": round(100 * (base - us) / base, 2)}
    print(json.dumps({"summary": summary}))


if __name__ == "__main__":
    main()
