"""Throughput of sampling from the trajectory model (paramgen.trajectory_sample_batch, mlpg_kernel in MODE_SAMPLE) on
the configs[1] batch of bench.py: 256 utterances of 500-700 frames, Merlin layout (D = 187, 62 smoothed output
columns and the copied vuv column), in float32 and float64, at n_samples 1, 4 and 16.

Each call is timed with CUDA events over windows of at least --window seconds of back-to-back calls, after warm-up,
alternating in the same process with mlpg_batch on the same inputs (the staged forward kernel); the reported time is
the median over --rounds windows.  Every call includes its one host synchronisation (the status word), as a user
sees it.  Reported:
  - sampled frames x smoothed columns per second, n_samples * frames * 62 / time;
  - the marginal time per extra sample, (t(16) - t(1)) / 15;
  - GB/s over algorithmic bytes: means and variances read once, the samples written once (the factor scratch that
    the sweeps re-read is not counted);
  - the max deviation of the scale = 0 output from mlpg_batch at the timed size.
The card name and power limit are printed with the numbers.

    python tools/bench_traj_sample.py [--rounds 5] [--window 1.0] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nnmnkwii_b200 import paramgen as G  # noqa: E402

WINDOWS = [(0, 0, np.array([1.0])), (1, 1, np.array([-0.5, 0.0, 0.5])), (1, 1, np.array([1.0, -2.0, 1.0]))]
N_SMOOTHED = 62


def batch(dtype, seed=0, n=256, mean_T=600):
    rng = np.random.default_rng(seed)
    lens = rng.integers(mean_T - 100, mean_T + 101, size=n)
    rows = int(lens.sum())
    m = np.cumsum(rng.standard_normal((rows, 187)), 0) * 0.01 + rng.standard_normal((rows, 187)) * 0.3
    v = rng.random((rows, 187)) + 0.1
    return lens, torch.from_numpy(m.astype(dtype)).cuda(), torch.from_numpy(v.astype(dtype)).cuda()


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name(0) + ", power limit not read, "
    return q


def window_ms(fn, seconds):
    """ms per call over a window of at least ``seconds`` of back-to-back calls, from CUDA events."""
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    e.synchronize()
    k = max(1, int(np.ceil(seconds * 1e3 / max(s.elapsed_time(e), 1e-3))))
    s.record()
    for _ in range(k):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_traj_sample needs a CUDA device")
    res = {"card": card(), "window_s": args.window, "rounds": args.rounds}
    print("card (name, power limit, max SM clock):", res["card"])
    layout = G.merlin_layout()
    for dtype in ("float32", "float64"):
        lens, m, v = batch(np.dtype(dtype))
        frames = int(lens.sum())
        es = m.element_size()
        kw = dict(lengths=lens, layout=layout)
        y = G.mlpg_batch(m, v, WINDOWS, **kw)
        dev0 = float((G.trajectory_sample_batch(m, v, WINDOWS, n_samples=2, scale=0.0, **kw) - y[None]).abs().max())
        fns = {"mlpg_batch": lambda: G.mlpg_batch(m, v, WINDOWS, **kw)}
        for n in (1, 4, 16):
            fns["sample_%d" % n] = (lambda n=n: G.trajectory_sample_batch(m, v, WINDOWS, n_samples=n, seed=n, **kw))
        for fn in fns.values():
            for _ in range(args.warmup):
                fn()
        torch.cuda.synchronize()
        times = {k: [] for k in fns}
        for _ in range(args.rounds):  # alternate the calls within every round
            for k, fn in fns.items():
                times[k].append(window_ms(fn, args.window))
        r = {"frames": frames, "utterances": len(lens), "scale0_max_abs_dev_from_mlpg_batch": dev0}
        for k, ts in times.items():
            ms = float(np.median(ts))
            n = int(k.split("_")[1]) if k.startswith("sample") else 1
            nbytes = (m.numel() + v.numel()) * es + n * frames * layout.D_out * es
            r[k] = {"ms": ms, "ms_spread": [float(min(ts)), float(max(ts))],
                    "frames_dims_per_s": n * frames * N_SMOOTHED / (ms * 1e-3),
                    "alg_GB_per_s": nbytes / (ms * 1e-3) / 1e9}
        r["marginal_ms_per_sample"] = (r["sample_16"]["ms"] - r["sample_1"]["ms"]) / 15.0
        res[dtype] = r
        print("%s: %d utterances, %d frames; scale = 0 vs mlpg_batch max |dev| = %.3g"
              % (dtype, len(lens), frames, dev0))
        for k in fns:
            print("  %-12s %8.3f ms  (%.3f-%.3f)  %.3g frames*dims/s  %6.1f GB/s"
                  % (k, r[k]["ms"], r[k]["ms_spread"][0], r[k]["ms_spread"][1], r[k]["frames_dims_per_s"],
                     r[k]["alg_GB_per_s"]))
        print("  marginal ms per extra sample: %.3f" % r["marginal_ms_per_sample"])
    line = json.dumps(res)
    print(line)
    if args.json:
        with open(args.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
