"""Throughput of the trajectory-model log-likelihood (paramgen.trajectory_log_likelihood_batch, and with its
gradients, the launch autograd.TrajectoryLogLikelihood makes) on the configs[1] batch of bench.py: 256 utterances of
about 600 frames, Merlin layout (D = 187), float32.

Compared on the same batch with mlpg_batch (one forward solve) and with autograd.MLPGBatch forward plus backward
(the training step that only reaches the means).  Host clock: the mean of synchronised repeated calls.  Device time:
the kernels' summed CUDA time per call from torch.profiler.  Algorithmic bytes per call: the means and variances
read once, the targets read once, and with the gradients the three gradient arrays written once.  The host
restatement (tests/traj_ll_oracle.py, banded) is timed on a few utterances for scale.

    python tools/bench_traj_ll.py [--steps 20] [--warmup 3] [--json out.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from nnmnkwii_b200 import autograd as A  # noqa: E402
from nnmnkwii_b200 import paramgen as G  # noqa: E402

WINDOWS = [(0, 0, np.array([1.0])), (1, 1, np.array([-0.5, 0.0, 0.5])), (1, 1, np.array([1.0, -2.0, 1.0]))]


def batch(seed=0, n=256, mean_T=600):
    rng = np.random.default_rng(seed)
    lens = rng.integers(mean_T - 100, mean_T + 101, size=n)
    rows = int(lens.sum())
    m = (np.cumsum(rng.standard_normal((rows, 187)), 0) * 0.01 + rng.standard_normal((rows, 187)) * 0.3)
    v = rng.random((rows, 187)) + 0.1
    x = np.cumsum(rng.standard_normal((rows, 63)), 0) * 0.01 + rng.standard_normal((rows, 63)) * 0.2
    to = lambda a: torch.from_numpy(a.astype(np.float32)).cuda()  # noqa: E731
    return lens, to(x), to(m), to(v)


def host_time(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps


def device_time(fn, steps):
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
        if t and ("mlpg" in e.key or "kernel" in e.key.lower()):
            total += t
            names[e.key[:90]] = t / steps
    return total / steps * 1e-6, names


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json")
    args = ap.parse_args()
    lens, x, m, v = batch()
    frames = int(lens.sum())
    layout = G.merlin_layout()
    kw = dict(lengths=lens, layout=layout)
    lay, padded, _ = G._traj_ll_check(x, m, v, WINDOWS, lens, None, layout)

    def ll_only():
        return G._traj_ll_device(x, m, v, WINDOWS, lens, None, lay, padded, False)

    def ll_grad():
        return G._traj_ll_device(x, m, v, WINDOWS, lens, None, lay, padded, True)

    def fwd():
        return G.mlpg_batch(m, v, WINDOWS, **kw)

    mg = m.clone().requires_grad_(True)
    go = torch.ones((frames, 187), dtype=torch.float32, device="cuda")  # single-stream MLPGBatch, D_out = 62 + 1

    def train_mlpg():
        y = A.mlpg_batch(mg[:, :180], v[:, :180], WINDOWS, lens)
        y.backward(go[:, :60])

    def train_tll():
        xg, mgg, vg = (t.detach().requires_grad_(True) for t in (x, m, v))
        A.trajectory_log_likelihood(xg, mgg, vg, WINDOWS, lens, layout).sum().backward()

    bytes_in = (m.numel() + v.numel() + x.numel()) * 4
    bytes_grad = bytes_in  # the three gradients, written once
    res = {"gpu": torch.cuda.get_device_name(0), "frames": frames, "utterances": len(lens)}
    for name, fn, nbytes in (("tll", ll_only, bytes_in), ("tll_grad", ll_grad, bytes_in + bytes_grad),
                             ("mlpg_batch", fwd, (m.numel() + v.numel() + frames * 63) * 4),
                             ("mlpgbatch_fwd_bwd_mgc", train_mlpg, None),
                             ("autograd_tll_fwd_bwd", train_tll, None)):
        t = host_time(fn, args.steps, args.warmup)
        dt, names = device_time(fn, max(3, args.steps // 4))
        res[name] = {"host_s": t, "device_s": dt, "frames_per_s": frames / t, "kernels": names}
        if nbytes:
            res[name]["alg_GB_per_s_device"] = nbytes / dt / 1e9 if dt else None
    # host restatement on a few utterances, for scale
    import traj_ll_oracle as O
    off = np.concatenate([[0], np.cumsum(lens)])
    xh, mh, vh = (a.cpu().numpy().astype(np.float64) for a in (x, m, v))
    t0 = time.perf_counter()
    n_host = 2
    for u in range(n_host):
        a, b = off[u], off[u + 1]
        O.log_likelihood(xh[a:b], mh[a:b], vh[a:b], WINDOWS, [(0, 60), (180, 1), (183, 1, "copy"), (184, 1)],
                         banded=True)
    th = (time.perf_counter() - t0) / n_host
    res["host_oracle"] = {"s_per_utterance": th, "frames_per_s": float(np.mean(lens[:n_host])) / th}
    line = json.dumps(res)
    print(line)
    if args.json:
        with open(args.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
