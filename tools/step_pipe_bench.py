"""Fast step kernel, classic vs. pipelined (QS_FAST_PIPE): µs per launch against the device's copy ceiling.

Prints the card (name, power limit, max SM clock), then the copy ceiling: a device-to-device copy with the step kernel's
read/write volume per launch of 65 536 drones (~27 MB read + ~26 MB written), rotated over buffers much larger than the 50 MB
L2 and timed with CUDA events.  Then it alternates the kernel variants (QS_FAST_PIPE=0: the classic one-tile-per-warp kernel,
4: the pipelined kernel, four tiles per warp), each in a fresh process, and times, in µs per launch:
  bench      the bench.py workload: 32 768 MultiHoverAviary x 2 drones, RPM, 8 batches rotating on one stream
  n262144    262 144 drones, 2 batches alternating
  n1048576   1 048 576 drones, 2 batches alternating
  graph      the bench launches replayed from a CUDA graph
  two_streams  even / odd batches on two streams
Each variant's bytes actually moved per launch over its time are printed against the ceiling.

    python tools/step_pipe_bench.py [--variants 0,4] [--runs 3] [--lib A=path ...]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D, A, B = 2, 4, 15
OBS = 12 + A * B
# bytes one drone-step actually moves in the fast kernel (DESIGN.md 4.1): float64 state r/w, action, the whole old row
# (bulk copy), the new row, per-aviary counter r/w + reward + three flags (per drone at D = 2)
ACT_BYTES = 104 + 104 + 16 + 4 * OBS + 4 * OBS + (4 + 4 + 4 + 3) / D


def card():
    try:
        q = "name,power.limit,clocks.max.sm"
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return dict(zip(q.split(","), [c.strip() for c in out.strip().split(",")]))
    except Exception as ex:  # noqa: BLE001
        return {"error": repr(ex)}


def copy_ceiling(torch, n_drones=65536, reps=2000, rot=8):
    """Device-to-device copy of the bytes one launch moves (half read, half written), over `rot` buffer pairs (> L2)."""
    dev = torch.device("cuda:0")
    nbytes = int(ACT_BYTES * n_drones / 2) // 256 * 256
    src = [torch.empty(nbytes // 4, dtype=torch.float32, device=dev).fill_(k) for k in range(rot)]
    dst = [torch.empty_like(s) for s in src]
    for k in range(3 * rot):
        dst[k % rot].copy_(src[k % rot])
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    res = []
    for _ in range(3):
        torch.cuda.synchronize()
        e0.record()
        for k in range(reps):
            dst[k % rot].copy_(src[k % rot])
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / reps
        res.append({"us_per_copy": round(us, 3), "tb_s": round(2 * nbytes / (us * 1e-6) / 1e12, 3)})
    out = {"bytes_read": nbytes, "bytes_written": nbytes, "runs": res, "tb_s": max(r["tb_s"] for r in res)}
    # the same mix without a launch boundary every 26 MB: one copy of all `rot` buffers at once
    big_s, big_d = torch.cat(src), torch.cat(dst)
    del src, dst
    for _ in range(3):
        big_d.copy_(big_s)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(50):
        big_d.copy_(big_s)
    e1.record()
    torch.cuda.synchronize()
    out["sustained_tb_s"] = round(2 * big_s.numel() * 4 * 50 / (e0.elapsed_time(e1) * 1e-3) / 1e12, 3)
    return out


def worker(steps):
    import torch
    from gym_pybullet_drones_b200.envs import MultiHoverAviary
    from gym_pybullet_drones_b200.utils.enums import ActionType, Physics
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(1234)
    out = {}

    def timed(fn, n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        fn(16)
        torch.cuda.synchronize()
        e0.record()
        fn(n)
        e1.record()
        torch.cuda.synchronize()
        return round(e0.elapsed_time(e1) * 1e3 / n, 3)

    R, E = 8, 65536 // D
    envs = [MultiHoverAviary(num_drones=D, physics=Physics.DYN, act=ActionType.RPM, num_envs=E, device=dev, autoreset="same_step",
                             host_copy=False) for _ in range(R)]
    acts = [[torch.rand((E, D, A), device=dev, generator=gen) * 2 - 1 for _ in range(16)] for _ in range(R)]
    for e in envs:
        e.reset()

    def run(n):
        for k in range(n):
            envs[k % R].step(acts[k % R][(k // R) % 16])

    out["bench"] = timed(run, steps)
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        run(2 * R)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        run(2 * R)
    out["graph"] = round(timed(lambda n: [g.replay() for _ in range(n)], max(1, steps // (2 * R))) / (2 * R), 3)
    del g
    s_even, s_odd = torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)
    cur = torch.cuda.current_stream(dev)

    def run2(n):
        s_even.wait_stream(cur)
        s_odd.wait_stream(cur)
        for k in range(n):
            i = k % R
            with torch.cuda.stream(s_even if (i & 1) == 0 else s_odd):
                envs[i].step(acts[i][(k // R) % 16])
        cur.wait_stream(s_even)
        cur.wait_stream(s_odd)

    out["two_streams"] = timed(run2, steps)
    del envs, acts
    torch.cuda.empty_cache()
    for n in (262144, 1048576):
        big = [MultiHoverAviary(num_drones=D, physics=Physics.DYN, act=ActionType.RPM, num_envs=n // D, device=dev, autoreset="same_step",
                                host_copy=False) for _ in range(2)]
        ba = torch.rand((n // D, D, A), device=dev, generator=gen) * 2 - 1
        for b in big:
            b.reset()
        out["n%d" % n] = timed(lambda m: [big[k & 1].step(ba) for k in range(m)], max(40, steps * 65536 // n))
        del big, ba
        torch.cuda.empty_cache()
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--variants", default="0,4", help="QS_FAST_PIPE values, alternated")
    ap.add_argument("--lib", action="append", default=[], help="NAME=path: an extra variant running another libquadsim.so")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--worker", action="store_true")
    a = ap.parse_args()
    sys.path.insert(0, ROOT)
    if a.worker:
        worker(a.steps)
        return
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device")
    info = {"card": card(), "actual_bytes_per_drone_step": ACT_BYTES}
    info["copy_ceiling"] = copy_ceiling(torch)
    print(json.dumps(info), flush=True)
    ceiling = info["copy_ceiling"]["tb_s"]
    variants = [("pipe%s" % v, {"QS_FAST_PIPE": v}) for v in a.variants.split(",") if v] + \
               [(s.split("=", 1)[0], {"QS_LIBQUADSIM": os.path.abspath(s.split("=", 1)[1])}) for s in a.lib]
    res = {name: [] for name, _ in variants}
    for r in range(a.runs):
        for name, env in variants:
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", "--steps", str(a.steps)], env=dict(os.environ, **env),
                               capture_output=True, text=True, cwd=ROOT)
            if p.returncode != 0:
                print(json.dumps({"variant": name, "run": r, "error": p.stderr[-2000:]}), flush=True)
                continue
            row = json.loads(p.stdout.strip().splitlines()[-1])
            res[name].append(row)
            print(json.dumps({"variant": name, "run": r, "us_per_launch": row}), flush=True)
    summary = {}
    for name, rows in res.items():
        if not rows:
            continue
        s = {}
        for k in rows[0]:
            v = [x[k] for x in rows]
            n = 65536 if k in ("bench", "graph", "two_streams") else int(k[1:])
            s[k] = {"us": v, "spread_pct": round(100 * (max(v) - min(v)) / min(v), 2),
                    "tb_s": round(ACT_BYTES * n / (min(v) * 1e-6) / 1e12, 3), "of_ceiling": round(ACT_BYTES * n / (min(v) * 1e-6) / 1e12 / ceiling, 3)}
        summary[name] = s
    print(json.dumps({"summary": summary, "copy_ceiling_tb_s": ceiling, "card": info["card"]}))


if __name__ == "__main__":
    main()
