"""Measure the segment-level modulation-spectrum post-filter and its statistics on the GPU.

    python tools/bench_ms_segment.py [--reps R] [--B 512] [--D 59] [--L 50] [--ns 64,128] [--host-utts 8]

Workload: a padded CUDA batch of B utterances of U{200..2000} frames (seeded) and D = 59 columns (``mgc[:, 1:]`` of
a 59th-order mel-cepstrum), in float32 and float64, segment length L = 50 (250 ms at a 5 ms shift).  For each
dtype and n:
  * modspec_statistics(segment=L) and modspec_post_filter(segment=L): the median CUDA-event time of one call, and
    of the nnk_ms_segment launch alone (kernel-only device time: the statistics' temporary, or the filter's gain
    table, already on the device);
  * frames/s over the live frames, and GB/s of the filter kernel over its algorithmic bytes (read every live
    frame of x once, write all B * T_max frames of y once), with that rate's share of the H100 SXM data sheet's
    3.35 TB/s;
  * the utterance-level filter (segment=None) at n = 2048 on the same batch, call and kernel alone;
  * the host restatement oracle/ms_segment.py on the first --host-utts utterances (frames/s, host clock) and the
    largest difference from the GPU result relative to the largest value.
Prints the card name, power limit and SM clock beside the numbers and one JSON line at the end.
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
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_modspec import time_ms  # noqa: E402

HBM_TBS = 3.35  # H100 SXM data sheet, TB/s
N_UTT = 2048    # the utterance-level filter's n for the comparison: every utterance fits


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                               "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def corpus(rng, B, D, dt, noise):
    """Padded (B, T_max, D) batch and lengths: random walks plus white noise scaled by ``noise``."""
    lens = rng.integers(200, 2001, B)
    pad = np.zeros((B, int(lens.max()), D), dt)
    for b, L in enumerate(lens):
        pad[b, :L] = rng.standard_normal((L, D)).cumsum(0) * 0.1 + noise * rng.standard_normal((L, D))
    return pad, lens


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--B", type=int, default=512)
    ap.add_argument("--D", type=int, default=59)
    ap.add_argument("--L", type=int, default=50)
    ap.add_argument("--ns", default="64,128")
    ap.add_argument("--host-utts", type=int, default=8)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_ms_segment needs a CUDA device"
    import oracle.ms_segment as O
    from nnmnkwii_b200 import _lib
    from nnmnkwii_b200.postfilters import (_ms_table, _segment_counts, _segment_launch, modspec_post_filter,
                                           modspec_statistics)
    from nnmnkwii_b200.preprocessing.modspec import _launch
    L = args.L
    res = {"card": card(), "B": args.B, "D": args.D, "L": L}
    print("card, power limit, max / current SM clock:", res["card"])
    for dt in (np.float32, np.float64):
        name = np.dtype(dt).name
        rng = np.random.default_rng(0)
        pad, lens = corpus(rng, args.B, args.D, dt, 0.02)
        nat_pad, nat_lens = corpus(rng, args.B, args.D, dt, 0.2)
        B, T, D = pad.shape
        frames = int(lens.sum())
        res.update(frames=frames, T_max=T)
        xt = torch.from_numpy(pad).cuda()
        nt = torch.from_numpy(nat_pad).cuda()
        item = np.dtype(dt).itemsize
        algo_bytes = (frames + B * T) * D * item
        r = {}
        for n in [int(s) for s in args.ns.split(",")]:
            K = n // 2 + 1
            G = modspec_statistics(xt, n=n, lengths=lens, segment=L)
            Nat = modspec_statistics(nt, n=n, lengths=nat_lens, segment=L)
            stats_ms = time_ms(lambda: modspec_statistics(xt, n=n, lengths=lens, segment=L), args.reps)
            J = _segment_counts(lens, L)
            S = int(J.sum())
            tmp = torch.empty((S, D, K), dtype=xt.dtype, device="cuda")
            off = torch.as_tensor(np.concatenate([[0], np.cumsum(J)[:-1]]), device="cuda")
            stats_kern_ms = time_ms(lambda: _segment_launch(_lib.NNK_MSSEG_LOGPOWER, n, L, xt, None, tmp, B, T, D,
                                                            lens, off), args.reps)
            del tmp
            out = modspec_post_filter(xt, Nat, G, k=1.0, n=n, lengths=lens, segment=L)
            pf_ms = time_ms(lambda: modspec_post_filter(xt, Nat, G, k=1.0, n=n, lengths=lens, segment=L), args.reps)
            tab = torch.from_numpy(_ms_table(Nat, G, 1.0, K, D, dt)).cuda()
            buf = torch.empty_like(xt)
            pf_kern_ms = time_ms(lambda: _segment_launch(_lib.NNK_MSSEG_POSTFILTER, n, L, xt, tab, buf, B, T, D, lens),
                                 args.reps)
            assert torch.equal(buf, out)
            gbs = algo_bytes / (pf_kern_ms * 1e-3) / 1e9
            # the host restatement on a few utterances
            o = out.cpu().numpy()
            Nh, Gh = ([a.cpu().numpy() for a in st] for st in (Nat, G))
            t0 = time.perf_counter()
            host = [O.post_filter(pad[b, :lens[b]], Nh, Gh, 1.0, n, L) for b in range(args.host_utts)]
            host_s = time.perf_counter() - t0
            host_frames = int(lens[:args.host_utts].sum())
            diff = max(float(np.abs(o[b, :len(h)] - h).max()) for b, h in enumerate(host))
            scale = max(float(np.abs(h).max()) for h in host)
            r["n%d" % n] = {
                "segments": S, "statistics_ms": stats_ms, "statistics_kernel_ms": stats_kern_ms,
                "statistics_frames_per_s": frames / (stats_ms * 1e-3),
                "post_filter_ms": pf_ms, "post_filter_kernel_ms": pf_kern_ms,
                "post_filter_frames_per_s": frames / (pf_ms * 1e-3),
                "post_filter_kernel_frames_per_s": frames / (pf_kern_ms * 1e-3),
                "post_filter_kernel_GBps": gbs, "post_filter_kernel_share_of_hbm": gbs / (HBM_TBS * 1e3),
                "host_frames_per_s": host_frames / host_s, "max_rel_diff_vs_host": diff / scale}
            print("%s n=%d L=%d: statistics %.3f ms (kernel %.3f ms, %.3g frames/s) | post-filter %.3f ms (kernel "
                  "%.3f ms, %.3g frames/s, %.1f GB/s = %.1f%% of %.2f TB/s) | host %.3g frames/s | max rel diff %.2e"
                  % (name, n, L, stats_ms, stats_kern_ms, frames / (stats_ms * 1e-3), pf_ms, pf_kern_ms,
                     frames / (pf_kern_ms * 1e-3), gbs, 100 * gbs / (HBM_TBS * 1e3), HBM_TBS, host_frames / host_s,
                     diff / scale))
        # the utterance-level filter at n = 2048 on the same batch
        Gu = modspec_statistics(xt, n=N_UTT, lengths=lens)
        Nu = modspec_statistics(nt, n=N_UTT, lengths=nat_lens)
        utt_ms = time_ms(lambda: modspec_post_filter(xt, Nu, Gu, k=1.0, n=N_UTT, lengths=lens), args.reps)
        tab = torch.from_numpy(_ms_table(Nu, Gu, 1.0, N_UTT // 2 + 1, D, dt)).cuda()
        buf = torch.empty_like(xt)
        utt_kern_ms = time_ms(lambda: _launch(_lib.NNK_MS_POSTFILTER, N_UTT, xt, tab, buf, None, B, T, T, D, lens, 1.0,
                                              1.0 / N_UTT), args.reps)
        ugbs = algo_bytes / (utt_kern_ms * 1e-3) / 1e9
        r["utterance_n%d" % N_UTT] = {"post_filter_ms": utt_ms, "post_filter_kernel_ms": utt_kern_ms,
                                      "post_filter_kernel_frames_per_s": frames / (utt_kern_ms * 1e-3),
                                      "post_filter_kernel_GBps": ugbs}
        print("%s utterance level n=%d: post-filter %.3f ms (kernel %.3f ms, %.3g frames/s, %.1f GB/s)"
              % (name, N_UTT, utt_ms, utt_kern_ms, frames / (utt_kern_ms * 1e-3), ugbs))
        res[name] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
