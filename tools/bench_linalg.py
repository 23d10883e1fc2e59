"""Measure the util.linalg kernels (csrc/nnk_linalg.cu) on the GPU.

    python tools/bench_linalg.py [--quick]

cholesky_inv_banded: T in {500, 1000, 4000}, w in {3, 5}, B in {1, 64}, on diagonally dominant banded
factors.  Reported as ms per call and GB/s of the algorithmic bytes against the 3.35 TB/s HBM3 data
sheet: 16 T^2 bytes per matrix (g written to the lower triangle, 4 T^2, read back, 4 T^2, and the full
P written, 8 T^2; the band itself is a few T w bytes).

cholesky_inv: N in {128, 512, 2048}, B in {1, 16}, lower factors of M M^T / N + I / 2.  Reported as FP64
FLOP/s of the algorithmic 2 N^3 / 3 operations per matrix (dpotri's count) against the H100 SXM data
sheet's 34 TFLOP/s FP64 (67 with the FP64 tensor cores, which this kernel does not use).

Kernel times are the median of CUDA-event timings of the C ABI call (no Python wrapper, no status read)
after warm-up.  The host baselines, one matrix at a time on the CPU of the GPU machine: scipy's dpotri plus
the mirror for cholesky_inv, and the C restatement of the reference's recurrence (oracle/nnk_oracle.c) for
cholesky_inv_banded.  Prints the card name and power limit beside the numbers and one JSON line at the end.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HBM = 3.35e12
FP64 = 34e12


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


def host_ms(fn, reps):
    fn()
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t) / reps * 1e3


def banded_factor(rng, T, w):
    R = np.zeros((T, T))
    for j in range(1, w):
        i = np.arange(j, T)
        R[i, i - j] = rng.uniform(-0.5, 0.5, T - j)
    R[np.arange(T), np.arange(T)] = 1.0 + 0.5 * w + rng.random(T)
    return R


def dense_factor(rng, N):
    M = rng.standard_normal((N, N))
    return np.linalg.cholesky(M @ M.T / N + 0.5 * np.eye(N))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="fewer repetitions (a rehearsal, not a measurement)")
    args = ap.parse_args()
    import scipy.linalg
    import torch

    import oracle
    from nnmnkwii_b200 import _device as dev
    from nnmnkwii_b200 import _lib
    from nnmnkwii_b200.util import linalg
    dev.require_cuda()
    reps = 3 if args.quick else 20
    rng = np.random.default_rng(0)
    res = {"card": card(), "banded": [], "dense": []}
    print("card, power limit:", res["card"])
    st = dev.current_stream_ptr(torch.device("cuda"))
    status = torch.zeros(1, dtype=torch.int64, device="cuda")

    for T in (500, 1000, 4000):
        for w in (3, 5):
            R = banded_factor(rng, T, w)
            host = host_ms(lambda: oracle.cholesky_inv_banded(R, w), 1 if T > 1000 else 3)
            assert np.array_equal(linalg.cholesky_inv_banded(R, w), oracle.cholesky_inv_banded(R, w))
            for B in (1, 64):
                Rd = torch.from_numpy(R).cuda().expand(B, T, T).contiguous()
                P = torch.empty_like(Rd)
                ms = time_ms(lambda: _lib.lib.nnk_cholesky_inv_banded(Rd.data_ptr(), w, T, B, P.data_ptr(),
                                                                      status.data_ptr(), st), reps)
                gbs = 16.0 * T * T * B / (ms * 1e-3) / 1e9
                row = {"T": T, "w": w, "B": B, "ms": ms, "GB/s": gbs, "of_hbm": gbs * 1e9 / HBM,
                       "host_oracle_ms_per_matrix": host}
                res["banded"].append(row)
                print("cholesky_inv_banded T=%5d w=%d B=%3d  %9.3f ms  %7.1f GB/s (%.3f of 3.35 TB/s)   "
                      "oracle on the host %8.1f ms per matrix" % (T, w, B, ms, gbs, gbs * 1e9 / HBM, host))
                del Rd, P

    for N in (128, 512, 2048):
        L = dense_factor(rng, N)
        host = host_ms(lambda: linalg_host(L, scipy.linalg), 3 if N > 512 else 10)
        for B in (1, 16):
            Ld = torch.from_numpy(L).cuda().expand(B, N, N).contiguous()
            P = torch.empty_like(Ld)
            ms = time_ms(lambda: _lib.lib.nnk_cholesky_inv(Ld.data_ptr(), 1, N, B, P.data_ptr(), status.data_ptr(),
                                                           st), reps)
            flops = 2.0 * N ** 3 / 3 * B / (ms * 1e-3)
            row = {"N": N, "B": B, "ms": ms, "TFLOP/s": flops / 1e12, "of_fp64": flops / FP64,
                   "host_dpotri_ms_per_matrix": host}
            res["dense"].append(row)
            print("cholesky_inv        N=%5d     B=%3d  %9.3f ms  %7.3f TFLOP/s (%.3f of 34 TFLOP/s)   "
                  "dpotri + mirror on the host %8.2f ms per matrix" % (N, B, ms, flops / 1e12, flops / FP64, host))
            del Ld, P
    assert int(status.item()) == 0
    print(json.dumps(res))


def linalg_host(L, sla):
    inv, info = sla.lapack.dpotri(L, lower=True)
    return np.tril(inv) + np.tril(inv, -1).T


if __name__ == "__main__":
    main()
