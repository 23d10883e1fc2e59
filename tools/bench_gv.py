"""bench_gv.py -- parameter generation considering global variance (paramgen.mlpg_gv_batch) on one GPU.

    python tools/bench_gv.py [--steps 10] [--warmup 3] [--oracle-utts 2] [--out FILE]

Two workloads, inputs resident on the device, float32 I/O, per-frame variances, 3 windows:
  cfg2   256 utterances, T ~ U{540..660}, the 187-column Merlin layout (62 smoothed columns + vuv copied)
  T1000  256 utterances of T = 1000, one stream of static_dim = 60 (180 columns)
For each: frames/s of mlpg_gv_batch at n_iter = 0, 5, 20 next to mlpg_batch on the same data (CUDA events around
`steps` calls, each call one kernel launch plus its host-side tables, no status synchronisation), the
algorithmic bytes (means + variances in, trajectories out; the scratch the kernel keeps is not counted) over that
time against 3.35 TB/s, and the host restatement's (oracle/gv.py, float64 NumPy / SciPy) frames/s on a few
utterances.  The card's name and power limit are read in the same run; without a GPU the script fails.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

WINDOWS = [(0, 0, np.array([1.0])), (1, 1, np.array([-0.5, 0.0, 0.5])), (1, 1, np.array([1.0, -2.0, 1.0]))]
HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def card():
    import torch
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_and_max_sm_clock"] = q
    except Exception as e:  # noqa: BLE001
        info["power_limit_and_max_sm_clock"] = "not read (%s)" % e
    return info


def workload(name, rng):
    from nnmnkwii_b200 import paramgen as G
    if name == "cfg2":
        lens = rng.integers(540, 661, size=256)
        D, layout = 187, G.merlin_layout()
    else:
        lens = np.full(256, 1000)
        D, layout = 180, G.StreamLayout.single(180, 3)
    n = int(lens.sum())
    m = rng.random((n, D), dtype=np.float32)
    v = rng.random((n, D), dtype=np.float32) + np.float32(0.1)
    return lens, m, v, layout


def algo_bytes(lens, layout):
    """means + variances read for every smoothed chain's windows, copied columns read once; out written once."""
    n = int(np.sum(lens))
    ch = layout.chains
    smoothed = int(np.sum(ch["flags"] == 0))
    copied = int(np.sum(ch["flags"] != 0))
    return n * 4 * (2 * 3 * smoothed + copied + layout.D_out)


def time_calls(fn, steps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3 / steps


def oracle_rate(lens, m, v, layout, gm, gvv, n_utt):
    import oracle.gv as ogv
    off = np.concatenate([[0], np.cumsum(lens)])
    frames = 0
    t0 = time.perf_counter()
    for u in range(n_utt):
        a, b = off[u], off[u + 1]
        for s in range(len(layout.slices)):
            o0, o1 = layout.slices[s]
            chains = layout.chains[o0:o1]
            if chains["flags"][0]:
                continue
            c0, sd = int(chains["in_col"][0]), o1 - o0
            ogv.mlpg_gv(m[a:b, c0:c0 + 3 * sd], v[a:b, c0:c0 + 3 * sd], WINDOWS, gm[o0:o1], gvv[o0:o1], 20)
        frames += b - a
    return frames / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--oracle-utts", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_gv.py needs a CUDA device: not measured")
    from nnmnkwii_b200 import paramgen as G
    res = {"card": card(), "steps": args.steps, "warmup": args.warmup, "results": {}}
    rng = np.random.default_rng(2024)
    for name in ("cfg2", "T1000"):
        lens, m, v, layout = workload(name, rng)
        md, vd = torch.from_numpy(m).cuda(), torch.from_numpy(v).cuda()
        gv = G.global_variance(G.mlpg_batch(md, vd, WINDOWS, lengths=lens, layout=layout), lengths=lens)
        gm = 2.0 * gv.mean(0).cpu().numpy() + 1e-6  # pull every column towards twice its c_m variance
        gvv = (0.1 * gm) ** 2
        frames = int(lens.sum())
        nbytes = algo_bytes(lens, layout)
        r = {"frames": frames, "algorithmic_bytes": nbytes}
        calls = {"mlpg_batch": lambda: G.mlpg_batch(md, vd, WINDOWS, lengths=lens, layout=layout, check=False)}
        for it in (0, 5, 20):
            calls["mlpg_gv_batch n_iter=%d" % it] = (
                lambda it=it: G.mlpg_gv_batch(md, vd, WINDOWS, gm, gvv, lengths=lens, layout=layout, n_iter=it,
                                              check=False))
        for k, fn in calls.items():
            t = time_calls(fn, args.steps, args.warmup)
            r[k] = {"seconds_per_call": t, "frames_per_s": frames / t,
                    "algorithmic_bytes_per_s": nbytes / t, "share_of_3.35TBps": nbytes / t / HBM_BYTES_PER_S}
        r["oracle_frames_per_s (float64 NumPy/SciPy, n_iter=20, %d utterances)" % args.oracle_utts] = oracle_rate(
            lens, m, v, layout, gm, gvv, args.oracle_utts)
        res["results"][name] = r
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
