"""bench_ms_gen.py -- parameter generation considering the modulation spectrum (paramgen.mlpg_ms_batch) on one GPU.

    python tools/bench_ms_gen.py [--steps 10] [--warmup 3] [--oracle-utts 2] [--out FILE]

Two workloads, inputs resident on the device, float32 I/O, per-frame variances, 3 windows, DFT length n = 1024:
  cfg2   256 utterances, T ~ U{540..660}, the 187-column Merlin layout (62 smoothed columns + vuv copied), as
         tools/bench_gv.py
  T1000  one utterance of T = 1000, one stream of static_dim = 60 (180 columns)
For each: frames/s of mlpg_ms_batch at n_iter = 0, 5, 20 next to mlpg_batch and mlpg_gv_batch (n_iter = 20) on the
same data (CUDA events around `steps` calls, no status synchronisation); the launches of one call; the split of
one n_iter = 20 call between its kernels (torch.profiler: the forward MLPG, the first MS launch, the banded solves
and the trial launches); and the host restatement's (oracle/ms_gen.py, float64 NumPy / SciPy) frames/s on a few
utterances.  The card's name and power limit are read in the same run; without a GPU the script fails.

The segment level (mlpg_ms_batch(segment=L), n = 64, L = 50) adds the same rows on cfg2 and on
  long   32 utterances of T = 20 000, one stream of static_dim = 60 (180 columns): only the segment level runs it
with the host restatement (tests/ms_gen_segment_oracle.py) timed on `--oracle-chains` chains of one utterance.
"""
import argparse
import json
import os
import re
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.bench_gv import WINDOWS, card, time_calls  # noqa: E402

N = 1024
SEG_N, SEG_L = 64, 50


def workload(name, rng):
    from nnmnkwii_b200 import paramgen as G
    if name == "cfg2":
        lens = rng.integers(540, 661, size=256)
        D, layout = 187, G.merlin_layout()
    elif name == "long":
        lens = np.full(32, 20000)
        D, layout = 180, G.StreamLayout.single(180, 3)
    else:
        lens = np.array([1000])
        D, layout = 180, G.StreamLayout.single(180, 3)
    n = int(lens.sum())
    m = rng.random((n, D), dtype=np.float32)
    m[:, :60] += np.cumsum(rng.standard_normal((n, 60)), 0).astype(np.float32) * 0.05
    v = rng.random((n, D), dtype=np.float32) + np.float32(0.1)
    return lens, m, v, layout


def ms_statistics(rng, D_out):
    """Statistics of rough trajectories, so that the MS term pulls every column."""
    nat = rng.standard_normal((16, N, D_out)) * 0.3 + np.cumsum(rng.standard_normal((16, N, D_out)), 1) * 0.05
    s = np.log(np.maximum(np.abs(np.fft.rfft(nat, N, axis=1)) ** 2, np.finfo(np.float64).tiny))
    return s.mean(0), s.var(0) + 0.5


def segment_statistics(rng, D_out):
    """Segment-level statistics (n = SEG_N, L = SEG_L) of rough trajectories."""
    import oracle.ms_segment as oseg
    nat = rng.standard_normal((4, 2000, D_out)) * 0.3 + np.cumsum(rng.standard_normal((4, 2000, D_out)), 1) * 0.05
    mean, var = oseg.statistics(list(nat), SEG_N, SEG_L)
    return mean, var + 0.5


def kernel_split(fn):
    """Seconds of device time per kernel class in one call of ``fn``."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    split, count = {}, {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = e.name
        if re.search(r"ms_gen_segment_kernel<\d+, true>", name):
            k = "trial (ms_gen_segment_kernel<LOGN, true>)"
        elif re.search(r"ms_gen_segment_kernel<\d+, false>", name):
            k = "first gradient (ms_gen_segment_kernel<LOGN, false>)"
        elif re.search(r"ms_gen_kernel<\d+, true>", name):
            k = "trial (ms_gen_kernel<LOGN, true>)"
        elif re.search(r"ms_gen_kernel<\d+, false>", name):
            k = "first gradient (ms_gen_kernel<LOGN, false>)"
        elif re.search(r"\bmlpg_kernel<", name):
            k = "banded solve (nnk_mlpg_solve)"
        elif "mlpg" in name:
            k = "forward MLPG (nnk_mlpg_fwd)"
        else:
            k = "other (dtype casts, copies)"
        split[k] = split.get(k, 0.0) + e.device_time_total * 1e-6
        count[k] = count.get(k, 0) + 1
    return {k: {"seconds": split[k], "kernels": count[k]} for k in sorted(split)}


def oracle_rate(lens, m, v, layout, mm, mv, n_utt):
    import oracle.ms_gen as O
    off = np.concatenate([[0], np.cumsum(lens)])
    frames = 0
    t0 = time.perf_counter()
    for u in range(min(n_utt, len(lens))):
        a, b = off[u], off[u + 1]
        for s in range(len(layout.slices)):
            o0, o1 = layout.slices[s]
            chains = layout.chains[o0:o1]
            if chains["flags"][0]:
                continue
            c0, sd = int(chains["in_col"][0]), o1 - o0
            O.mlpg_ms(m[a:b, c0:c0 + 3 * sd].astype(np.float64), v[a:b, c0:c0 + 3 * sd].astype(np.float64),
                      WINDOWS, mm[:, o0:o1], mv[:, o0:o1], 20)
        frames += b - a
    return frames / (time.perf_counter() - t0)


def segment_oracle_rate(lens, m, v, layout, mm, mv, n_chains):
    """Frames/s of the host restatement of the segment level, from ``n_chains`` chains of the first utterance."""
    import ms_gen_segment_oracle as S
    T = int(lens[0])
    smoothed = [i for i in range(len(layout.chains)) if not layout.chains["flags"][i]][:n_chains]
    t0 = time.perf_counter()
    for i in smoothed:
        ch = layout.chains[i]
        cols = [int(ch["in_col"]) + w * int(ch["win_stride"]) for w in range(3)]
        o = int(ch["out_col"])
        S.mlpg_ms(m[:T, cols].astype(np.float64), v[:T, cols].astype(np.float64), WINDOWS, mm[:, o:o + 1],
                  mv[:, o:o + 1], SEG_L, 20)
    per_chain = (time.perf_counter() - t0) / len(smoothed)
    return T / (per_chain * int(np.sum(layout.chains["flags"] == 0)))


def run_segment(r, lens, md, vd, m, v, layout, rng, args):
    """Segment-level rows of one workload into ``r``."""
    import torch
    from nnmnkwii_b200 import _lib
    from nnmnkwii_b200 import paramgen as G
    mm, mv = segment_statistics(rng, layout.D_out)
    frames = int(lens.sum())
    for it in (0, 5, 20):
        fn = (lambda it=it: G.mlpg_ms_batch(md, vd, WINDOWS, mm, mv, lengths=lens, layout=layout, n_iter=it,
                                            check=False, segment=SEG_L))
        t = time_calls(fn, args.steps, args.warmup)
        n0 = _lib.launch_count()
        fn()
        key = "mlpg_ms_batch segment=%d n=%d n_iter=%d" % (SEG_L, SEG_N, it)
        r[key] = {"seconds_per_call": t, "frames_per_s": frames / t, "launches": _lib.launch_count() - n0}
    torch.cuda.synchronize()
    split = kernel_split(lambda: G.mlpg_ms_batch(md, vd, WINDOWS, mm, mv, lengths=lens, layout=layout, n_iter=20,
                                                 check=False, segment=SEG_L))
    r["kernel split of one segment-level n_iter=20 call"] = split
    r["per trial (segment level, n_iter=20)"] = {
        k: split[k]["seconds"] / 20 for k in split if k.startswith(("trial", "banded solve"))}
    r["segment oracle_frames_per_s (float64 NumPy/SciPy, n_iter=20, from %d chains)" % args.oracle_chains] = (
        segment_oracle_rate(lens, m, v, layout, mm, mv, args.oracle_chains))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--oracle-utts", type=int, default=2)
    ap.add_argument("--oracle-chains", type=int, default=2)
    ap.add_argument("--only", default=None, help="comma-separated workloads (cfg2, T1000, long)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_ms_gen.py needs a CUDA device: not measured")
    from nnmnkwii_b200 import _lib
    from nnmnkwii_b200 import paramgen as G
    res = {"card": card(), "n": N, "steps": args.steps, "warmup": args.warmup, "results": {}}
    rng = np.random.default_rng(2024)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    names = args.only.split(",") if args.only else ["cfg2", "T1000", "long"]
    for name in ("cfg2", "T1000", "long"):
        # the segment-level rows draw from their own generators: the utterance-level rows keep their inputs
        lens, m, v, layout = workload(name, np.random.default_rng(2025) if name == "long" else rng)
        if name not in names:
            continue
        md, vd = torch.from_numpy(m).cuda(), torch.from_numpy(v).cuda()
        r = {"utterances": len(lens), "frames": int(lens.sum())}
        if name == "long":  # the utterance level refuses T > 4096: segment rows only, next to mlpg_batch
            t = time_calls(lambda: G.mlpg_batch(md, vd, WINDOWS, lengths=lens, layout=layout, check=False),
                           args.steps, args.warmup)
            r["mlpg_batch"] = {"seconds_per_call": t, "frames_per_s": r["frames"] / t}
            run_segment(r, lens, md, vd, m, v, layout, np.random.default_rng(2026), args)
            res["results"][name] = r
            continue
        mm, mv = ms_statistics(rng, layout.D_out)
        gv = G.global_variance(G.mlpg_batch(md, vd, WINDOWS, lengths=lens, layout=layout), lengths=lens)
        gm = 2.0 * gv.mean(0).cpu().numpy() + 1e-6
        gvv = (0.1 * gm) ** 2
        frames = int(lens.sum())
        calls = {"mlpg_batch": lambda: G.mlpg_batch(md, vd, WINDOWS, lengths=lens, layout=layout, check=False),
                 "mlpg_gv_batch n_iter=20": lambda: G.mlpg_gv_batch(md, vd, WINDOWS, gm, gvv, lengths=lens,
                                                                    layout=layout, n_iter=20, check=False)}
        for it in (0, 5, 20):
            calls["mlpg_ms_batch n_iter=%d" % it] = (
                lambda it=it: G.mlpg_ms_batch(md, vd, WINDOWS, mm, mv, lengths=lens, layout=layout, n_iter=it,
                                              check=False))
        for k, fn in calls.items():
            t = time_calls(fn, args.steps, args.warmup)
            r[k] = {"seconds_per_call": t, "frames_per_s": frames / t}
        for it in (0, 5, 20):
            n0 = _lib.launch_count()
            G.mlpg_ms_batch(md, vd, WINDOWS, mm, mv, lengths=lens, layout=layout, n_iter=it, check=False)
            r["mlpg_ms_batch n_iter=%d" % it]["launches"] = _lib.launch_count() - n0
        r["kernel split of one mlpg_ms_batch n_iter=20 call"] = kernel_split(
            lambda: G.mlpg_ms_batch(md, vd, WINDOWS, mm, mv, lengths=lens, layout=layout, n_iter=20, check=False))
        r["oracle_frames_per_s (float64 NumPy/SciPy, n_iter=20, %d utterances)" % min(args.oracle_utts, len(lens))] = (
            oracle_rate(lens, m, v, layout, mm, mv, args.oracle_utts))
        if name == "cfg2":
            run_segment(r, lens, md, vd, m, v, layout, np.random.default_rng(2026), args)
        res["results"][name] = r
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
