"""Measure the waveform / F0 preprocessing kernels on the GPU.

    python tools/bench_wave.py [--quick]

Workloads (signals built by tiling the golden speech window at seeded gains, so the inverse filter's
speculation sees speech statistics):
  W1  configs[1] scale: 256 signals of U{540..660} frames x 80 samples (16 kHz, 5 ms frames)
  W2  configs[4] scale: 8192 signals of U{200..2000} frames x 80, a padded float32 CUDA batch with lengths
  W3  one 16 kHz signal of one hour (57.6 M samples)
For preemphasis / inv_preemphasis at coef 0.97: median CUDA-event time after warm-up, GB/s on 8 B per
valid sample (float32 in and out) and its share of the 3.35 TB/s data-sheet bandwidth; the repair
counters (also at 0.86, 0.99, 0.999 on W1); scipy's lfilter on one host core for W1.  Also mulaw_quantize
on W2 and interp1d on the golden lf0 column at configs[1] and configs[4] frame counts.  Prints the card
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
HBM = 3.35e12


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


def signals(audio, n, lo, hi, rng, fixed=None):
    """A padded float32 CUDA batch (built on the device: W2 is 5 GB) and its lengths."""
    import torch
    lens = fixed if fixed is not None else rng.integers(lo, hi + 1, n) * 80
    Tmax = int(lens.max())
    base = torch.from_numpy(np.tile(audio, Tmax // len(audio) + 2).astype(np.float32)).cuda()
    x = torch.zeros((n, Tmax), dtype=torch.float32, device="cuda")
    for b in range(n):
        off = int(rng.integers(0, len(audio)))
        x[b, :lens[b]] = base[off:off + lens[b]] * float(rng.uniform(0.1, 1.5))
    return x, lens


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="W2 at 1/8 scale (rehearsal)")
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_wave needs a CUDA device"
    from scipy import signal

    from nnmnkwii_b200 import preprocessing as P
    from nnmnkwii_b200.preprocessing import waveform
    g = np.load(os.path.join(ROOT, "tests", "golden", "wave_reference_golden.npz"))
    audio = g["audio"] / 32768.0
    rng = np.random.default_rng(0)
    res = {"card": card()}
    print("card, power limit:", res["card"])
    n2 = 1024 if args.quick else 8192
    x1, l1 = signals(audio, 256, 540, 660, rng)
    x2, l2 = signals(audio, n2, 200, 2000, rng)
    x3, l3 = signals(audio, 1, 0, 0, rng, fixed=np.array([57_600_000]))
    for name, xt, lens in (("W1", x1, l1), ("W2", x2, l2), ("W3", x3, l3)):
        lt = None if name == "W3" else lens
        n = int(lens.sum())
        for fn in ("preemphasis", "inv_preemphasis"):
            f = getattr(P, fn)
            ms = time_ms(lambda: f(xt, 0.97, lengths=lt), args.reps)
            gbs = 8.0 * n / (ms * 1e-3) / 1e9
            r = {"ms": ms, "GB/s": gbs, "share": gbs * 1e9 / HBM, "floor_ms": 8.0 * n / HBM * 1e3, "samples": n}
            if fn == "inv_preemphasis":
                r["repair"] = waveform._repair_counters()
            res["%s_%s" % (fn, name)] = r
            print("%-16s %s %10d samples %9.3f ms %8.1f GB/s share %.3f floor %.3f ms %s"
                  % (fn, name, n, ms, gbs, r["share"], r["floor_ms"], r.get("repair", "")))
    x1t = x1
    for c in (0.86, 0.99, 0.999):
        ms = time_ms(lambda: P.inv_preemphasis(x1t, c, lengths=l1), 5, warmup=1)
        res["inv_W1_%g" % c] = {"ms": ms, "repair": waveform._repair_counters()}
        print("inv_preemphasis W1 coef %g: %.3f ms, repair (chunks, samples) %s" % (c, ms, waveform._repair_counters()))
    t0 = time.perf_counter()
    b, a = np.array([1.0], np.float32), np.array([1.0, -0.97], np.float32)
    for row, n in zip(x1.cpu().numpy(), l1):
        signal.lfilter(b, a, row[:n])
    res["scipy_lfilter_W1_s"] = time.perf_counter() - t0
    print("scipy lfilter (one host core) W1: %.3f s" % res["scipy_lfilter_W1_s"])
    del x3
    x2t = x2.clamp_(-1, 1)
    ms = time_ms(lambda: P.mulaw_quantize(x2t), args.reps)
    nb = x2.numel() * (4 + 8)
    res["mulaw_quantize_W2"] = {"ms": ms, "GB/s": nb / (ms * 1e-3) / 1e9, "share": nb / (ms * 1e-3) / HBM}
    print("mulaw_quantize W2 (padded %d samples): %.3f ms %.1f GB/s share %.3f"
          % (x2.numel(), ms, nb / (ms * 1e-3) / 1e9, nb / (ms * 1e-3) / HBM))
    lf0 = np.concatenate([g["lf0_%d" % i] for i in range(3)])
    for name, B, lo, hi in (("configs[1]", 256, 540, 660), ("configs[4]", 8192, 200, 2000)):
        lens = rng.integers(lo, hi + 1, B)
        T = int(lens.max())
        f = np.zeros((B, T), np.float32)
        for i in range(B):
            off = int(rng.integers(0, len(lf0) - T)) if len(lf0) > T else 0
            seg = np.tile(lf0, T // len(lf0) + 2)[off:off + T]
            f[i] = seg
        ft = torch.from_numpy(f).cuda()
        ms = time_ms(lambda: P.interp1d(ft, "slinear", lengths=lens), args.reps)
        res["interp1d_" + name] = {"ms": ms, "frames": int(lens.sum())}
        print("interp1d slinear %s: %d frames %.3f ms" % (name, int(lens.sum()), ms))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
