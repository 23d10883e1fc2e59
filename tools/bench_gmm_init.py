"""Time the k-means initialisation of baseline.gmm.GaussianMixture on the host (scikit-learn) and on the device
(csrc/nnk_kmeans.cu) on the two workloads of tools/bench_gmm.py.

    python tools/bench_gmm_init.py [--workloads aligner,vc] [--reps 3]

Per workload one JSON line: the host KMeans(n_init=1) wall seconds; the device initialisation wall seconds (host
clock, ending in a synchronise); seeding and Lloyd ms from CUDA events, n_iter and us per Lloyd iteration; the
algorithmic bytes (N D sizeof(x) per pass) and FP64 FLOP (2 N K D) of one iteration with the larger of the two
H100 SXM data-sheet bounds named; whole-fit wall seconds with init_device False and True, alternated in the same
run; whether the labels are equal; the card name and power limit, read in the same call.
"""
import argparse
import json
import os
import sys
import time
import warnings

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_gmm import aligner_matrix, card, vc_matrix  # noqa: E402

PEAK_FP64 = 34e12
PEAK_HBM = 3.35e12


def run(name, X, K, reps):
    import torch
    from sklearn.cluster import KMeans
    from sklearn.utils import check_random_state

    from nnmnkwii_b200 import _lib
    from nnmnkwii_b200.baseline import gmm as G
    N, D = X.shape
    X64 = X.astype(np.float64)
    t0 = time.perf_counter()
    ref = KMeans(n_clusters=K, n_init=1, random_state=check_random_state(0)).fit(X64)
    t_host = time.perf_counter() - t0

    Xd = torch.from_numpy(X).cuda()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        G._device_kmeans(Xd, K, random_state=0)  # warm-up: module load, first launches
        walls = []
        for _ in range(reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            labels, _, _, n_iter = G._device_kmeans(Xd, K, random_state=0)
            torch.cuda.synchronize()
            walls.append(time.perf_counter() - t0)

        # the phases with CUDA events: seeding, then the Lloyd iterations (status read-backs included)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        st = G._KMeansState(Xd, K, centre=True)
        first, u = G._kmeans_plusplus_draws(N, K, check_random_state(0))
        ev[0].record()
        st.prepare()
        st.seed(first, u)
        ev[1].record()
        tol_abs = float(st.read_status()[_lib.NNK_KM_VAR_MEAN]) * 1e-4
        it = 0
        for it in range(1, 301):
            st.lloyd(True)
            s = st.read_status()
            if s[_lib.NNK_KM_EMPTY] > 0:
                st.relocate_empty_clusters()
                st.average()
                s = st.read_status()
            if s[_lib.NNK_KM_CHANGED] == 0 or s[_lib.NNK_KM_SHIFT] <= tol_abs:
                break
        ev[2].record()
        ev[2].synchronize()
        seed_ms, lloyd_ms = ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2])

        fits = {False: [], True: []}
        for _ in range(reps):
            for flag in (False, True):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                G.GaussianMixture(n_components=K, random_state=0, init_device=flag).fit(X)
                fits[flag].append(time.perf_counter() - t0)

    bytes_pass = N * D * X.itemsize
    flop = 2.0 * N * K * D
    rec = {
        "workload": name, "N": int(N), "D": int(D), "K": int(K), "dtype": str(X.dtype),
        "host_kmeans_s": round(t_host, 4),
        "device_init_wall_s_median": round(float(np.median(walls)), 5),
        "speedup_host_over_device": round(t_host / float(np.median(walls)), 1),
        "seeding_ms": round(seed_ms, 3), "lloyd_ms": round(lloyd_ms, 3), "n_iter": int(n_iter),
        "us_per_lloyd_iter": round(1e3 * lloyd_ms / max(1, it), 2),
        "bytes_per_pass": bytes_pass, "fp64_flop_per_iter": flop,
        "hbm_bound_us": round(1e6 * bytes_pass / PEAK_HBM, 2), "fp64_bound_us": round(1e6 * flop / PEAK_FP64, 2),
        "bound": "memory" if bytes_pass / PEAK_HBM > flop / PEAK_FP64 else "fp64",
        "fit_wall_s_host_init_median": round(float(np.median(fits[False])), 4),
        "fit_wall_s_device_init_median": round(float(np.median(fits[True])), 4),
        "labels_equal": bool(np.array_equal(labels.cpu().numpy(), ref.labels_)),
        "n_iter_equal": bool(n_iter == ref.n_iter_),
    }
    print(json.dumps(rec), flush=True)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="aligner,vc")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch
    torch.cuda.set_device(0)
    name, plim = card()
    print(json.dumps({"card": name, "power_limit": plim}), flush=True)
    for w in args.workloads.split(","):
        if w == "aligner":
            run("aligner_configs3", aligner_matrix(), 16, args.reps)
        elif w == "vc":
            run("vc_72x64", vc_matrix(), 64, args.reps)
        else:
            raise SystemExit("unknown workload %r" % w)


if __name__ == "__main__":
    main()
