"""bench_mix_gen.py -- parameter generation from per-frame mixtures (paramgen.mlpg_mixture_batch) on one GPU.

    python tools/bench_mix_gen.py [--steps 5] [--warmup 2] [--oracle-utts 2] [--out FILE]

Workload at acoustic-model scale: 256 utterances of 1000 frames in the 187-column Merlin layout (63 output
columns), per-frame mixtures with M = 1, 4 and 8 components as CUDA tensors (what an MDN head hands over), float32
and float64.  For each (dtype, M):
  * frames/s of mlpg_mixture_batch at n_iter = 0 (the most-probable collapse) and n_iter = 5, wall clock of whole
    calls (each ends with its one synchronisation), and of mlpg_batch on the same batch's (T, 187) rows;
  * from a separate torch.profiler run of one n_iter = 5 call: device time of the SELECT launch, of one E-step
    launch and of one MLPG solve (every kernel the solves launch, over the 6 solves);
  * the E-step's algorithmic bytes, computed here from the shapes: means and variances of every component
    (itemsize of the input), the log-normaliser table (8 bytes per component and frame), the trajectory rows
    (8 * 63 per frame) and the E and V rows written (2 * 8 * 187 per frame); over the E-step time that is its
    rate, and over 3.35 TB/s (the H100 SXM data sheet's HBM3 bandwidth) its share of it.
The float64 NumPy / SciPy restatement (tests/mix_gen_oracle.py) runs on a few utterances (M = 4, n_iter = 5).
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
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

WINDOWS = [(0, 0, np.array([1.0])), (1, 1, np.array([-0.5, 0.0, 0.5])), (1, 1, np.array([1.0, -2.0, 1.0]))]
MERLIN = [(0, 60), (180, 1), (183, 1, "copy"), (184, 1)]
N_UTT, T_UTT, D_IN, D_OUT = 256, 1000, 187, 63
HBM_BYTES_PER_S = 3.35e12


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


def batch(M, dtype, seed):
    """Per-frame mixtures on the device: smooth component means, log-weights of comparable size."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    n = N_UTT * T_UTT
    lw = torch.randn((n, M), generator=g, device="cuda", dtype=torch.float64) * 0.5
    mu = torch.randn((n, M, D_IN), generator=g, device="cuda", dtype=torch.float64) * 0.1
    mu += torch.randn((1, M, D_IN), generator=g, device="cuda", dtype=torch.float64)
    s2 = torch.rand((n, M, D_IN), generator=g, device="cuda", dtype=torch.float64) * 0.5 + 0.1
    return [a.to(dtype) for a in (lw, mu, s2)]


def profile_call(fn):
    """Device seconds of (SELECT launch, one E-step launch, one solve) in one n_iter = 5 call."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    select = estep = solve = 0.0
    n_estep = 0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if "mix_gen_kernel" in e.key:
            mode = int(e.key.split("mix_gen_kernel<")[1].split(",")[1])
            if mode == 0:
                select += t
            elif mode == 1:
                estep += t
                n_estep += e.count
        elif e.key.startswith(("void nnk::", "nnk::")) or "mlpg" in e.key:
            solve += t
    return select * 1e-6, estep * 1e-6 / max(n_estep, 1), solve * 1e-6 / 6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--oracle-utts", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_mix_gen.py measures on the GPU"
    import mix_gen_oracle as O
    from nnmnkwii_b200 import paramgen as G
    layout = G.merlin_layout()
    lens = [T_UTT] * N_UTT
    frames = N_UTT * T_UTT
    lines = [{"card": card()}]
    for dtype in (torch.float32, torch.float64):
        for M in (1, 4, 8):
            lw, mu, s2 = batch(M, dtype, M)
            call = {k: (lambda k=k: G.mlpg_mixture_batch(lw, mu, s2, WINDOWS, lengths=lens, layout=layout, n_iter=k))
                    for k in (0, 5)}
            t0 = timed(call[0], args.steps, args.warmup)
            t5 = timed(call[5], args.steps, args.warmup)
            rows_mu, rows_s2 = mu[:, 0].contiguous(), s2[:, 0].contiguous()
            t_mlpg = timed(lambda: G.mlpg_batch(rows_mu, rows_s2, WINDOWS, lengths=lens, layout=layout),
                           args.steps, args.warmup)
            t_sel, t_e, t_solve = profile_call(call[5])
            item = mu.element_size()
            nbytes = frames * (2 * M * D_IN * item + 8 * M + 8 * D_OUT + 2 * 8 * D_IN)
            lines.append({
                "workload": "%d utts x %d frames, Merlin layout (187 -> 63), M = %d, %s" % (
                    N_UTT, T_UTT, M, str(dtype).replace("torch.", "")),
                "frames_per_s_n_iter_0": frames / t0,
                "frames_per_s_n_iter_5": frames / t5,
                "em_iteration_s_wall": (t5 - t0) / 5,
                "mlpg_batch_frames_per_s": frames / t_mlpg,
                "select_kernel_s": t_sel,
                "estep_kernel_s": t_e,
                "estep_bytes": nbytes,
                "estep_bytes_per_s": nbytes / t_e if t_e > 0 else None,
                "estep_share_of_3_35_TB_s": nbytes / t_e / HBM_BYTES_PER_S if t_e > 0 else None,
                "solve_kernels_s": t_solve,
            })
            del lw, mu, s2, rows_mu, rows_s2
            torch.cuda.empty_cache()
    rng = np.random.default_rng(0)
    k = args.oracle_utts
    utts = []
    for _ in range(k):
        lw = rng.standard_normal((T_UTT, 4)) * 0.5
        mu = rng.standard_normal((T_UTT, 4, D_IN)) * 0.1 + rng.standard_normal((1, 4, D_IN))
        utts.append((lw, mu, rng.random((T_UTT, 4, D_IN)) * 0.5 + 0.1))
    t = time.perf_counter()
    for u in utts:
        O.mlpg_mixture(*u, WINDOWS, 5, streams=MERLIN)
    lines.append({"oracle": "tests/mix_gen_oracle.py, Merlin layout, M = 4, n_iter = 5, %d utterances" % k,
                  "oracle_frames_per_s": k * T_UTT / (time.perf_counter() - t)})
    text = "\n".join(json.dumps(x) for x in lines)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
