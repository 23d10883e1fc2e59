"""bench_gmm_traj_em.py -- trajectory EM of GMM voice conversion (baseline.gmm.MLPG.transform_em_batch) on one GPU.

    python tools/bench_gmm_traj_em.py [--steps 5] [--warmup 2] [--n-iter 5] [--oracle-utts 1] [--out FILE]

Workload at voice-conversion scale: 64 utterances of 600 frames, 24 static dimensions + delta (D = 48), a
synthetic joint GMM with M = 32 and M = 64 mixtures, source frames from the host (as users call it).  For each M:
  * frames/s of transform_batch (the arg-max-mixture conversion, c_0) and of transform_em_batch at n_iter;
  * frames/s per EM iteration: (time(n_iter) - time(0)) / n_iter, wall clock of whole calls (each ends with its
    one synchronisation);
  * the float64 NumPy / SciPy restatement (oracle/gmm_traj_em.py) per EM iteration on a few utterances;
  * from a separate torch.profiler run: device time per iteration of the E-step kernel (gmm_traj_em_kernel)
    and of the MLPG solve (every other kernel a call launches per iteration), and the E-step's FP64 FMA rate
    (T M D^2 FMAs for the affine maps).
The card's name and power limit are read in the same run; without a GPU the script fails.
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

WINDOWS = [(0, 0, np.array([1.0])), (1, 1, np.array([-0.5, 0.0, 0.5]))]
N_UTT, T_UTT, STATIC = 64, 600, 24


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


def joint_gmm(rng, M, dim):
    import types
    A = rng.standard_normal((M, 2 * dim, 2 * dim)) / np.sqrt(2 * dim)
    cov = A @ A.transpose(0, 2, 1) + 0.5 * np.eye(2 * dim)
    w = rng.random(M) + 0.1
    return types.SimpleNamespace(means_=rng.standard_normal((M, 2 * dim)), covariances_=cov, weights_=w / w.sum(),
                                 covariance_type="full")


def timed(fn, steps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) / steps


def profile_iteration(m, srcs, n_iter, out_dir):
    """Device time per EM iteration of the E-step kernel and of everything else the iterations launch, from the
    difference of a call at n_iter and at 0 iterations."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    def kernel_times(k):
        m.transform_em_batch(srcs, n_iter=k)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            m.transform_em_batch(srcs, n_iter=k)
            torch.cuda.synchronize()
        estep = other = 0.0
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", None)
            if t is None:
                t = e.cuda_time_total
            if e.key.startswith(("void nnk::", "nnk::")) or "_kernel" in e.key:
                if "gmm_traj_em_kernel" in e.key:
                    estep += t
                else:
                    other += t
        if out_dir:
            prof.export_chrome_trace(os.path.join(out_dir, "gmm_traj_em_M%d_n%d.pt.trace.json" % (m.num_mixtures, k)))
        return estep * 1e-6, other * 1e-6
    e1, o1 = kernel_times(n_iter)
    e0, o0 = kernel_times(0)
    return (e1 - e0) / n_iter, (o1 - o0) / n_iter


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--n-iter", type=int, default=5)
    ap.add_argument("--oracle-utts", type=int, default=1)
    ap.add_argument("--out", default=None)
    ap.add_argument("--trace-dir", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_gmm_traj_em.py measures on the GPU"
    import oracle.gmm_traj_em as OT
    from nnmnkwii_b200.baseline.gmm import MLPG
    lines = [{"card": card()}]
    frames = N_UTT * T_UTT
    for M in (32, 64):
        rng = np.random.default_rng(M)
        D = STATIC * len(WINDOWS)
        g = joint_gmm(rng, M, D)
        m = MLPG(g, windows=WINDOWS)
        srcs = [rng.standard_normal((T_UTT, D)) for _ in range(N_UTT)]
        t_map = timed(lambda: m.transform_batch(srcs), args.steps, args.warmup)
        t_em0 = timed(lambda: m.transform_em_batch(srcs, n_iter=0), args.steps, args.warmup)
        t_em = timed(lambda: m.transform_em_batch(srcs, n_iter=args.n_iter), args.steps, args.warmup)
        per_iter = (t_em - t_em0) / args.n_iter
        k = args.oracle_utts
        t = time.perf_counter()
        OT.transform_em(g, WINDOWS, srcs[0], 0)
        t0 = time.perf_counter() - t
        t = time.perf_counter()
        for s in srcs[:k]:
            OT.transform_em(g, WINDOWS, s, 1)
        t_or = (time.perf_counter() - t) / k - t0
        e_dev, o_dev = profile_iteration(m, srcs, args.n_iter, args.trace_dir)
        fma = frames * M * D * D
        lines.append({
            "workload": "%d utts x %d frames, D = %d (24 static + delta), M = %d" % (N_UTT, T_UTT, D, M),
            "transform_batch_frames_per_s": frames / t_map,
            "transform_em_batch_n_iter": args.n_iter,
            "transform_em_batch_frames_per_s": frames / t_em,
            "em_iteration_s": per_iter,
            "em_iteration_frames_per_s": frames / per_iter,
            "oracle_em_iteration_frames_per_s": T_UTT / t_or,
            "estep_kernel_s_per_iteration": e_dev,
            "mlpg_kernels_s_per_iteration": o_dev,
            "estep_fp64_fma_per_s": fma / e_dev if e_dev > 0 else None,
        })
    text = "\n".join(json.dumps(x) for x in lines)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
