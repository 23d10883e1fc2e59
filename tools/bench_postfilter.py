"""Time the Merlin post-filter kernels (csrc/nnk_postfilter.cu) on two seeded workloads.

    python tools/bench_postfilter.py [--iters 50] [--no-exp-lib PATH | --no-phase-split] [--cpu-frames 200]

D = 60, alpha = 0.41, fftlen = 1024, minimum_phase_order = 511, float32 frames on the device:
(a) cfg1: the configs[1] batch of bench.py, 256 utterances of T ~ U{540..660} (about 1.5e5 frames);
(b) cfg4: the configs[4] scale, 8192 utterances of T ~ U{200..2000} (about 9.0e6 frames), as one call.
Per workload it prints one JSON line: the median CUDA-event time of `postfilter_kernel` per call over
--iters launches, frames/s, and the FP64 rate of the GEMM, 4 (L/2 + 1) D flops per frame, against the
H100 SXM data-sheet peaks (34 TFLOP/s FP64, 67 TFLOP/s FP64 tensor core).  The exponential phase is split
off by timing the same launches with a library built with -DNNK_PF_NO_EXP (exp replaced by one FMA; its
results are wrong), which this script compiles into a temporary directory unless --no-exp-lib names one.
The basis build (`postfilter_basis_kernel`) is timed on its own line, and the CPU restatement of the
chain (oracle/sptk_postfilter.py: numpy, float64, literal SPTK loops -- not pysptk) on a third.
The card name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_FP64 = 34e12
PEAK_FP64_TC = 67e12
D, ALPHA, FFTLEN, ORDER = 60, 0.41, 1024, 511


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        idx = os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0] or "0"
        out = subprocess.run(["nvidia-smi", "-i", idx, "--query-gpu=power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        out = "unknown (%s)" % type(e).__name__
    return name, out


def workloads():
    cfg1 = int(np.random.default_rng(1234).integers(540, 661, size=256).sum())
    cfg4 = int(np.random.default_rng(4242).integers(200, 2001, size=8192).sum())
    return {"cfg1": cfg1, "cfg4": cfg4}


def time_kernels(iters):
    """{workload: median ms of one postfilter_apply launch} and the median ms of one basis build."""
    import torch

    from nnmnkwii_b200 import _lib
    from nnmnkwii_b200 import _device as dev

    torch.cuda.set_device(0)
    st = dev.current_stream_ptr(torch.device("cuda", 0))
    L = _lib.lib
    n = int(L.nnk_postfilter_basis_elems(D, FFTLEN))
    basis = torch.empty(n, dtype=torch.float64, device="cuda")
    w = torch.full((D,), 1.4, dtype=torch.float64, device="cuda")
    w[:2] = 1.0

    def events(fn, reps):
        ts = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            ts.append(a.elapsed_time(b))
        return float(np.median(ts))

    def build():
        _lib.check(L.nnk_postfilter_basis(ALPHA, D, ORDER, FFTLEN, basis.data_ptr(), n, st), "basis")

    build()
    torch.cuda.synchronize()
    basis_ms = events(build, 20)
    res = {}
    g = torch.Generator(device="cuda").manual_seed(0)
    for name, N in workloads().items():
        x = torch.randn((N, D), generator=g, device="cuda", dtype=torch.float32) * (
            0.8 / (1.0 + torch.arange(D, device="cuda", dtype=torch.float32)))
        out = torch.empty_like(x)

        def run():
            _lib.check(L.nnk_postfilter_apply(x.data_ptr(), _lib.NNK_F32, N, D, D, w.data_ptr(), FFTLEN,
                                              basis.data_ptr(), n, out.data_ptr(), D, st), "apply")

        for _ in range(3):
            run()
        torch.cuda.synchronize()
        reps = max(5, iters if N < 1_000_000 else iters // 5)
        res[name] = (N, events(run, reps))
        del x, out
        torch.cuda.empty_cache()
    return res, basis_ms


def build_no_exp(tmp):
    code = ("import sys; sys.path.insert(0, %r); from nnmnkwii_b200 import build as B; B.OBJ = %r; B.LIB = %r; "
            "B.NVCC_FLAGS = B.NVCC_FLAGS + ['-DNNK_PF_NO_EXP']; B.build()"
            % (ROOT, os.path.join(tmp, "obj"), os.path.join(tmp, "libnnk_b200.so")))
    subprocess.check_call([sys.executable, "-c", code])
    return os.path.join(tmp, "libnnk_b200.so")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--no-exp-lib", default=None, help="a libnnk_b200.so built with -DNNK_PF_NO_EXP")
    ap.add_argument("--no-phase-split", action="store_true")
    ap.add_argument("--cpu-frames", type=int, default=200)
    ap.add_argument("--kernels-only", action="store_true", help=argparse.SUPPRESS)  # child run of the phase split
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_postfilter: no CUDA device (these are GPU timings; there is no CPU fallback)")
    if args.kernels_only:
        res, _ = time_kernels(args.iters)
        print(json.dumps({k: v[1] for k, v in res.items()}))
        return
    name, power = card()
    res, basis_ms = time_kernels(args.iters)
    no_exp = {}
    if not args.no_phase_split:
        with tempfile.TemporaryDirectory(prefix="nnk_pf_noexp_") as tmp:
            lib = args.no_exp_lib or build_no_exp(tmp)
            env = dict(os.environ, NNK_LIB_PATH=lib)
            out = subprocess.run([sys.executable, os.path.abspath(__file__), "--kernels-only", "--iters", str(args.iters)],
                                 env=env, capture_output=True, text=True, check=True).stdout
            no_exp = json.loads(out.strip().splitlines()[-1])
    flops_per_frame = 4 * (FFTLEN // 2 + 1) * D
    for wl, (N, ms) in res.items():
        rate = flops_per_frame * N / (ms * 1e-3)
        line = {
            "workload": wl, "frames": N, "D": D, "alpha": ALPHA, "fftlen": FFTLEN, "order": ORDER, "dtype": "float32",
            "kernel_ms": round(ms, 4), "frames_per_s": N / (ms * 1e-3),
            "gemm_fp64_flops_per_s": rate, "share_of_fp64_34T": rate / PEAK_FP64, "share_of_fp64_tc_67T": rate / PEAK_FP64_TC,
            "gpu": name, "power_limit": power,
        }
        if wl in no_exp:
            line["kernel_ms_without_exp"] = round(no_exp[wl], 4)
            line["exp_phase_ms"] = round(ms - no_exp[wl], 4)
        print(json.dumps(line))
    print(json.dumps({"basis_build_ms": round(basis_ms, 4), "D": D, "fftlen": FFTLEN, "order": ORDER, "gpu": name,
                      "power_limit": power}))
    from oracle import sptk_postfilter as P
    x = np.random.default_rng(0).standard_normal((args.cpu_frames, D)) * (0.8 / (1.0 + np.arange(D)))
    t = time.perf_counter()
    P.merlin_post_filter(x, ALPHA, ORDER, FFTLEN)
    dt = time.perf_counter() - t
    print(json.dumps({"cpu_restatement": "oracle/sptk_postfilter.py (numpy float64, literal SPTK loops; not pysptk)",
                      "frames": args.cpu_frames, "seconds": round(dt, 3), "frames_per_s": args.cpu_frames / dt}))


if __name__ == "__main__":
    main()
