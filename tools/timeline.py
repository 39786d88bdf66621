"""Per-warp phase timeline of the fast step kernel (tools, not product): builds a -DQS_TIMELINE copy of the library
(build/libquadsim_timeline.so, %globaltimer stamps by lane 0 of every warp), runs the bench workload and prints where a
warp's time goes.  Stamps: 0 start, 1 after the readiness wait (per-warp ticket, and griddepcontrol.wait when kept), 2 loads issued / bulk copy issued (once the state loads
have arrived), 3 physics done, 4 state stored, 5 old span arrived, 6 bulk store + terminal rows issued, 7 exit.
The pipelined kernel (A = 4 unless QS_FAST_PIPE=0) stamps per 32-drone tile: 0 its warp started, 1 its loads issued (after its
readiness), 2 tile started (its state and actions in registers), 3 physics done, 4 state stored, 5 old span arrived, 6 bulk store + terminal rows issued, 7 published.

    python tools/timeline.py --build          # here (nvcc)
    python tools/timeline.py [--act ONE_D_RPM] [--n 65536]   # on the GPU box
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
LIB = os.path.join(ROOT, "build", "libquadsim_timeline.so")


def build():
    from gym_pybullet_drones_b200 import _native as N
    N.build()
    obj = os.path.join(ROOT, "build", "obj", "step_fast_timeline.o")
    nvcc = "nvcc"
    subprocess.run([nvcc] + N.NVCC_FLAGS + ["-DQS_TIMELINE", "-c", "-o", obj, os.path.join(ROOT, "gym_pybullet_drones_b200", "csrc", "step_fast.cu")], check=True)
    objs = [os.path.join(N.OBJ_DIR, os.path.splitext(os.path.basename(s))[0] + ".o") for s in N.SOURCES if not s.endswith("step_fast.cu")] + [obj]
    subprocess.run([nvcc, "-shared"] + N.ARCH + ["-o", LIB] + objs, check=True)
    print("built", LIB)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--build", action="store_true")
    ap.add_argument("--act", default="RPM")
    ap.add_argument("--n", type=int, default=65536)
    ap.add_argument("--isolated", action="store_true", help="sync + L2 scrub before the sampled launch")
    a = ap.parse_args()
    if a.build:
        build()
        return
    os.environ["QS_LIBQUADSIM"] = LIB
    import numpy as np
    import torch
    from gym_pybullet_drones_b200 import _native as N
    from gym_pybullet_drones_b200.envs import MultiHoverAviary
    from gym_pybullet_drones_b200.utils.enums import ActionType, Physics
    dev = torch.device("cuda:0")
    D, n = 2, a.n
    A = 4 if a.act == "RPM" else 1
    R = 8 if n <= 65536 else 2
    envs = [MultiHoverAviary(num_drones=D, physics=Physics.DYN, act=ActionType[a.act], num_envs=n // D, autoreset="same_step") for _ in range(R)]
    g = torch.Generator(device=dev).manual_seed(0)
    acts = [torch.rand((n // D, D, A), device=dev, generator=g) * 2 - 1 for _ in envs]
    for e in envs:
        e.reset()
    for k in range(64):
        envs[k % R].step(acts[k % R])
    torch.cuda.synchronize()
    L = N.lib()
    nw = min(n // 32, 8192)

    def fetch(slot):
        b = np.zeros(nw * 16, np.uint64)
        rc = L.qs_debug_timeline(b.ctypes.data_as(C.c_void_p), C.c_int(nw * 16), C.c_int(slot))
        assert rc == 0, rc
        return b.reshape(nw, 16).astype(np.int64)

    if a.isolated:
        scrub = torch.empty(192 << 20, dtype=torch.uint8, device=dev)
        scrub.fill_(1)
        torch.cuda.synchronize()
        L.qs_debug_set_slot(1)
        envs[0].step(acts[0])
    else:
        for k in range(24):
            L.qs_debug_set_slot(k & 3)
            envs[k % R].step(acts[k % R])
    torch.cuda.synchronize()
    gaps = None
    if not a.isolated:      # consecutive launches 20..23 live in slots 0..3: gap = first release of launch k+1 - last exit of launch k
        tl = [fetch(sl) for sl in range(4)]
        last = [int(max(x[:, k].max() for k in range(16))) for x in tl]
        gaps = {"last_exit_to_next_release_us": [round((int(tl[k + 1][:, 1].min()) - last[k]) / 1e3, 2) for k in range(3)],
                "release_to_release_us": [round((int(tl[k + 1][:, 1].min()) - int(tl[k][:, 1].min())) / 1e3, 2) for k in range(3)],
                "next_first_start_minus_last_exit_us": [round((int(tl[k + 1][:, 0].min()) - last[k]) / 1e3, 2) for k in range(3)]}
    t = fetch(1 if a.isolated else 3)
    used = [k for k in range(16) if (t[:, k] > 0).all()]
    t = t[:, used]
    t0 = t[:, 0].min()
    rel = (t - t0) / 1e3            # us since the first warp started
    all_names = ["start", "after_pdl_wait", "state_arrived", "physics_done", "derived", "task_done", "state_stored", "span_stored/arrived", "rows_done", "exit"]
    if a.act == "RPM" and os.environ.get("QS_FAST_PIPE") != "0":     # step_pipe_kernel: one row per 32-drone tile
        all_names = ["warp_start", "loads_issued", "tile_start", "physics_done", "state_stored", "span_arrived", "span_store_issued", "published"]
    names = [all_names[k] if k < len(all_names) else "s%d" % k for k in used]
    out = {"act": a.act, "n": n, "isolated": a.isolated, "env": {k: v for k, v in os.environ.items() if k.startswith("QS_") and k != "QS_LIBQUADSIM"}, "warps": nw, "phases_us": {}}
    for k, nm in enumerate(names):
        c = rel[:, k]
        out["phases_us"][nm] = {"min": round(float(c.min()), 2), "p10": round(float(np.percentile(c, 10)), 2), "median": round(float(np.median(c)), 2),
                                "p90": round(float(np.percentile(c, 90)), 2), "max": round(float(c.max()), 2)}
    d = np.diff(rel, axis=1)
    out["per_warp_durations_us_median"] = {names[k] + "->" + names[k + 1]: round(float(np.median(d[:, k])), 2) for k in range(len(names) - 1)}
    out["span_us"] = round(float(rel[:, -1].max()), 2)
    out["gaps"] = gaps
    out["release_to_last_exit_us"] = round(float(rel[:, -1].max() - rel[:, 1].min()), 2)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
