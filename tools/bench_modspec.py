"""Measure modulation-spectrum smoothing on the GPU against the host NumPy path.

    python tools/bench_modspec.py [--reps R] [--B 32] [--D 60]

Workload: a padded float32 / float64 CUDA batch of B utterances of U{200..1500} frames (seeded) and D feature
columns, n = 4096, modfs = 200, cutoff = 50, log domain, norm None: the defaults of modspec_smoothing on 5 ms
frames.  For each dtype: the median CUDA-event time of one batched modspec_smoothing call after warm-up, of
modspec with the phase, and of the ModSpecBatch forward + backward; the host path (per utterance numpy.fft
rfft, log-power band removal and irfft, on the utterance arrays already in host memory) timed with a host
clock; and the largest difference between the two results relative to the largest value.  Prints the card
name and power limit beside the numbers and one JSON line at the end.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
N, MODFS, CUTOFF = 4096, 200, 50


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def time_ms(fn, reps, warmup=3):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def host_smoothing(x):
    """Log-power band removal of one (T, D) utterance with numpy.fft, the host path users run today."""
    T = len(x)
    X = np.fft.rfft(x, n=N, axis=0)
    keep = int(N * CUTOFF / MODFS) + 1
    mag = np.abs(X)
    unit = np.where(mag > 0, X / np.where(mag > 0, mag, 1), 1)
    X[keep:] = unit[keep:]  # log power 0: unit amplitude, phase kept
    return np.fft.irfft(X, n=N, axis=0)[:T]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--B", type=int, default=32)
    ap.add_argument("--D", type=int, default=60)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_modspec needs a CUDA device"
    from nnmnkwii_b200 import autograd as A
    from nnmnkwii_b200 import preprocessing as P
    rng = np.random.default_rng(0)
    lens = rng.integers(200, 1501, args.B)
    T = int(lens.max())
    frames = int(lens.sum())
    res = {"card": card(), "B": args.B, "D": args.D, "n": N, "frames": frames, "T_max": T}
    print("card, power limit:", res["card"])
    print("B=%d D=%d n=%d frames=%d (T in [%d, %d])" % (args.B, args.D, N, frames, lens.min(), lens.max()))
    for dt in (np.float32, np.float64):
        name = np.dtype(dt).name
        utts = [(rng.standard_normal((L, args.D)).cumsum(0) * 0.1).astype(dt) for L in lens]
        pad = np.zeros((args.B, T, args.D), dt)
        for b, u in enumerate(utts):
            pad[b, :len(u)] = u
        xt = torch.from_numpy(pad).cuda()
        out = P.modspec_smoothing(xt, MODFS, n=N, cutoff=CUTOFF, lengths=lens)
        gpu_ms = time_ms(lambda: P.modspec_smoothing(xt, MODFS, n=N, cutoff=CUTOFF, lengths=lens), args.reps)
        ms_ms = time_ms(lambda: P.modspec(xt, n=N, return_phase=True, lengths=lens), args.reps)
        yt = xt.clone().requires_grad_(True)

        def fwd_bwd():
            A.modspec_batch(yt, lens, N).sum().backward()
        grad_ms = time_ms(fwd_bwd, args.reps)
        host = []
        t0 = time.perf_counter()
        for u in utts:
            host.append(host_smoothing(u))
        host_s = time.perf_counter() - t0
        o = out.cpu().numpy()
        diff = max(float(np.abs(o[b, :len(h)] - h).max()) for b, h in enumerate(host))
        scale = max(float(np.abs(h).max()) for h in host)
        r = {"smoothing_ms": gpu_ms, "modspec_with_phase_ms": ms_ms, "modspec_fwd_bwd_ms": grad_ms,
             "host_numpy_smoothing_ms": host_s * 1e3, "speedup_vs_host": host_s * 1e3 / gpu_ms,
             "max_rel_diff_vs_host": diff / scale}
        res[name] = r
        print("%s: modspec_smoothing %.3f ms | modspec+phase %.3f ms | ModSpecBatch fwd+bwd %.3f ms | "
              "host numpy smoothing %.1f ms (%.0fx) | max rel diff %.2e"
              % (name, gpu_ms, ms_ms, grad_ms, host_s * 1e3, host_s * 1e3 / gpu_ms, diff / scale))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
