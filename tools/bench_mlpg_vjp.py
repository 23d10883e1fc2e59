"""Throughput of the gradient of MLPG in its means and variances (paramgen.mlpg_vjp_batch, mlpg_kernel in MODE_VJP,
and the forward plus backward of autograd.MLPGWithVariances) on the configs[1] batch of bench.py: 256 utterances of
500-700 frames, Merlin layout (D = 187, 62 smoothed output columns and the copied vuv column), in float32 and float64.

Alternating in the same process, on the same inputs:
  - mlpg_vjp_batch: one MODE_VJP launch and its status-word synchronisation;
  - MLPGWithVariances forward (mlpg_batch) + backward (mlpg_vjp_batch);
  - MLPGBatch forward + backward, the MGE step that reaches the means only, on the single mgc stream (the only
    layout MLPGBatch takes);
  - mlpg_grad_batch alone (the means-only backward, Merlin layout);
  - the trajectory log-likelihood with its three gradients (the MODE_TLL_GRAD launch).
Host time: a host clock around --steps back-to-back calls that ends in a device synchronise, the median over --rounds
rounds.  Device time: the kernels' summed CUDA time per call from torch.profiler, in a run of its own after the
timing rounds.  Algorithmic bytes of the VJP: means, variances and grad_output read once, both gradients written once
(the factor scratch is not counted); GB/s are over device time.  The card name and power limit are read in the same
process as the timings and printed with them.

    python tools/bench_mlpg_vjp.py [--rounds 5] [--steps 20] [--warmup 3] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nnmnkwii_b200 import autograd as A  # noqa: E402
from nnmnkwii_b200 import paramgen as G  # noqa: E402

WINDOWS = [(0, 0, np.array([1.0])), (1, 1, np.array([-0.5, 0.0, 0.5])), (1, 1, np.array([1.0, -2.0, 1.0]))]


def batch(dtype, seed=0, n=256, mean_T=600):
    rng = np.random.default_rng(seed)
    lens = rng.integers(mean_T - 100, mean_T + 101, size=n)
    rows = int(lens.sum())
    m = np.cumsum(rng.standard_normal((rows, 187)), 0) * 0.01 + rng.standard_normal((rows, 187)) * 0.3
    v = rng.random((rows, 187)) + 0.1
    go = rng.standard_normal((rows, 63))
    x = np.cumsum(rng.standard_normal((rows, 63)), 0) * 0.01 + rng.standard_normal((rows, 63)) * 0.2
    return (lens,) + tuple(torch.from_numpy(a.astype(dtype)).cuda() for a in (m, v, go, x))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name(0) + ", power limit not read, "
    return q


def host_ms(fn, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3


def device_ms(fn, steps):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    total, names = 0.0, {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if t and e.device_type is not None and "cuda" in str(e.device_type).lower():
            total += t
            names[e.key[:90]] = t / steps * 1e-3
    return total / steps * 1e-3, names


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mlpg_vjp needs a CUDA device")
    res = {"card": card(), "rounds": args.rounds, "steps": args.steps}
    print("card (name, power limit, max SM clock):", res["card"])
    layout = G.merlin_layout()
    for dtype in ("float32", "float64"):
        lens, m, v, go, x = batch(np.dtype(dtype))
        frames = int(lens.sum())
        es = m.element_size()
        kw = dict(lengths=lens, layout=layout)
        lay, padded, _ = G._traj_ll_check(x, m, v, WINDOWS, lens, None, layout)
        mg, vg = m.clone().requires_grad_(True), v.clone().requires_grad_(True)
        mgc_m, mgc_v = m[:, :180].contiguous().requires_grad_(True), v[:, :180].contiguous()
        go_mgc = go[:, :60].float().contiguous()

        def vjp():
            return G.mlpg_vjp_batch(m, v, WINDOWS, go, **kw)

        def with_variances():
            mg.grad = vg.grad = None
            A.mlpg_with_variances(mg, vg, WINDOWS, lens, layout).backward(go)

        def mlpgbatch_mgc():
            mgc_m.grad = None
            A.mlpg_batch(mgc_m, mgc_v, WINDOWS, lens).backward(go_mgc)

        def grad_batch():
            return G.mlpg_grad_batch(v, WINDOWS, go, lens, layout=layout)

        def tll_grad():
            return G._traj_ll_device(x, m, v, WINDOWS, lens, None, lay, padded, True)

        fns = {"mlpg_vjp_batch": vjp, "mlpg_with_variances_fwd_bwd": with_variances,
               "mlpgbatch_mgc_fwd_bwd": mlpgbatch_mgc, "mlpg_grad_batch": grad_batch, "tll_grad": tll_grad}
        for fn in fns.values():
            for _ in range(args.warmup):
                fn()
        torch.cuda.synchronize()
        times = {k: [] for k in fns}
        for _ in range(args.rounds):  # alternate the calls within every round
            for k, fn in fns.items():
                times[k].append(host_ms(fn, args.steps))
        r = {"frames": frames, "utterances": len(lens)}
        vjp_bytes = (2 * m.numel() + 2 * v.numel() + go.numel()) * es
        for k, fn in fns.items():
            dms, names = device_ms(fn, max(3, args.steps // 4))
            ms = float(np.median(times[k]))
            r[k] = {"host_ms": ms, "host_ms_spread": [float(min(times[k])), float(max(times[k]))],
                    "device_ms": dms, "kernels_ms": names}
            if k == "mlpg_vjp_batch":
                r[k]["alg_GB_per_s_device"] = vjp_bytes / (dms * 1e-3) / 1e9 if dms else None
        res[dtype] = r
        print("%s: %d utterances, %d frames" % (dtype, len(lens), frames))
        for k in fns:
            extra = ("  %6.1f GB/s (device)" % r[k]["alg_GB_per_s_device"]) if "alg_GB_per_s_device" in r[k] else ""
            print("  %-28s host %8.3f ms (%.3f-%.3f)  device %8.3f ms%s"
                  % (k, r[k]["host_ms"], r[k]["host_ms_spread"][0], r[k]["host_ms_spread"][1], r[k]["device_ms"],
                     extra))
            for name, t in sorted(r[k]["kernels_ms"].items(), key=lambda a: -a[1])[:3]:
                print("      %8.3f ms  %s" % (t, name))
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if args.json:
        with open(args.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
