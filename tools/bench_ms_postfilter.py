"""Measure the modulation-spectrum post-filter and its statistics on the GPU against the host NumPy restatement.

    python tools/bench_ms_postfilter.py [--reps R] [--B 32] [--D 60] [--B-stats 512]

Workload (that of tools/bench_modspec.py): a padded CUDA batch of B utterances of U{200..1500} frames (seeded) and
D feature columns, n = 4096, in float32 and float64.  For each dtype:
  * the median CUDA-event time of one batched modspec_post_filter call (host statistics, k = 1), which includes
    the float64 (a, c) table the host builds and uploads on every call; the host clock time of building that
    table; and the CUDA-event time of the nnk_modspec launch alone with the table already on the device;
  * modspec_smoothing on the same batch (the same two FFTs per column), for comparison;
  * modspec_statistics on a corpus of B-stats utterances drawn the same way;
  * the host path: oracle/ms_postfilter.py (numpy.fft, float64) per utterance, timed with a host clock, and the
    largest difference between the two results relative to the largest value.
Prints the card name and power limit beside the numbers and one JSON line at the end.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_modspec import card, time_ms  # noqa: E402

N, MODFS, CUTOFF = 4096, 200, 50


def corpus(rng, B, D, dt, smooth):
    """Padded (B, T_max, D) batch and lengths: random walks plus white noise, the noise scaled by ``smooth``."""
    lens = rng.integers(200, 1501, B)
    pad = np.zeros((B, int(lens.max()), D), dt)
    for b, L in enumerate(lens):
        pad[b, :L] = rng.standard_normal((L, D)).cumsum(0) * 0.1 + smooth * rng.standard_normal((L, D))
    return pad, lens


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--B", type=int, default=32)
    ap.add_argument("--D", type=int, default=60)
    ap.add_argument("--B-stats", type=int, default=512)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_ms_postfilter needs a CUDA device"
    import oracle.ms_postfilter as O
    from nnmnkwii_b200 import _lib
    from nnmnkwii_b200 import preprocessing as P
    from nnmnkwii_b200.postfilters import _ms_table, modspec_post_filter, modspec_statistics
    from nnmnkwii_b200.preprocessing.modspec import _launch
    res = {"card": card(), "B": args.B, "D": args.D, "n": N, "B_stats": args.B_stats}
    print("card, power limit:", res["card"])
    for dt in (np.float32, np.float64):
        name = np.dtype(dt).name
        rng = np.random.default_rng(0)
        pad, lens = corpus(rng, args.B, args.D, dt, 0.02)
        nat_pad, nat_lens = corpus(rng, args.B, args.D, dt, 0.2)
        res.update(frames=int(lens.sum()), T_max=int(lens.max()))
        xt = torch.from_numpy(pad).cuda()
        G = modspec_statistics(pad, n=N, lengths=lens)
        Nat = modspec_statistics(nat_pad, n=N, lengths=nat_lens)
        out = modspec_post_filter(xt, Nat, G, k=1.0, n=N, lengths=lens)
        pf_ms = time_ms(lambda: modspec_post_filter(xt, Nat, G, k=1.0, n=N, lengths=lens), args.reps)
        # the host part of a call: range checks and the float64 (a, c) table
        B, T, D = xt.shape
        ts = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            table = _ms_table(Nat, G, 1.0, N // 2 + 1, D, dt)
            ts.append(time.perf_counter() - t0)
        table_ms = float(np.median(ts)) * 1e3
        # the launch alone, the table already on the device
        tab = torch.from_numpy(table).cuda()
        buf = torch.empty_like(xt)
        kern_ms = time_ms(lambda: _launch(_lib.NNK_MS_POSTFILTER, N, xt, tab, buf, None, B, T, T, D, lens, 1.0,
                                          1.0 / N), args.reps)
        assert torch.equal(buf, out)
        sm_ms = time_ms(lambda: P.modspec_smoothing(xt, MODFS, n=N, cutoff=CUTOFF, lengths=lens), args.reps)
        spad, slens = corpus(np.random.default_rng(1), args.B_stats, args.D, dt, 0.02)
        st = torch.from_numpy(spad).cuda()
        stats_ms = time_ms(lambda: modspec_statistics(st, n=N, lengths=slens), max(5, args.reps // 5))
        del st
        host = []
        t0 = time.perf_counter()
        for b, L in enumerate(lens):
            host.append(O.post_filter(pad[b, :L], Nat, G, 1.0, N))
        host_s = time.perf_counter() - t0
        o = out.cpu().numpy()
        diff = max(float(np.abs(o[b, :len(h)] - h).max()) for b, h in enumerate(host))
        scale = max(float(np.abs(h).max()) for h in host)
        r = {"post_filter_ms": pf_ms, "post_filter_kernel_ms": kern_ms, "host_table_ms": table_ms,
             "smoothing_ms": sm_ms, "statistics_ms": stats_ms, "host_numpy_post_filter_ms": host_s * 1e3,
             "speedup_vs_host": host_s * 1e3 / pf_ms, "max_rel_diff_vs_host": diff / scale}
        res[name] = r
        print("%s: modspec_post_filter %.3f ms (launch alone %.3f ms, host table %.3f ms) | modspec_smoothing "
              "%.3f ms | modspec_statistics B=%d %.3f ms | host numpy post-filter %.1f ms (%.0fx) | max rel diff %.2e"
              % (name, pf_ms, kern_ms, table_ms, sm_ms, args.B_stats, stats_ms, host_s * 1e3, host_s * 1e3 / pf_ms,
                 diff / scale))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
