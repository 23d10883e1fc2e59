"""Time the device EM of baseline.gmm.GaussianMixture (csrc/nnk_gmm_em.cu) on two seeded workloads.

    python tools/bench_gmm.py [--iters 10] [--workloads aligner,vc] [--no-sklearn]

(a) aligner: configs[3]-style pairs (512 pairs, T ~ 800, 25-dim MFCC-like) -> one FastDTW pass (melcd) ->
    the joint (N * L_max, 50) matrix IterativeDTWAligner fits, K = 16;
(b) vc: about 2e5 frames of D = 72 joint static + delta features, K = 64.
Per workload it prints one JSON line: median device ms per EM iteration (CUDA events) split into the E-step
and the M-step + factorisation, the achieved FP64 rate 2 N K D (D + 1) / t against the H100 SXM data-sheet
peaks (34 TFLOP/s FP64, 67 TFLOP/s FP64 tensor core), the host initialisation (k-means) wall time, the
wall time of a whole fit (max_iter=100), and scikit-learn's seconds per iteration on the same host, timed
over two iterations started from the device fit's parameters.  The card name and power limit are read
in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time
import warnings

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PEAK_FP64 = 34e12
PEAK_FP64_TC = 67e12


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


def aligner_matrix(seed=0, n_pairs=512, T=800, D=25):
    from nnmnkwii_b200.metrics import melcd
    from nnmnkwii_b200.preprocessing.alignment import DTWAligner
    rng = np.random.default_rng(seed)
    X = np.zeros((n_pairs, T, D), np.float32)
    Y = np.zeros((n_pairs, T, D), np.float32)
    for i in range(n_pairs):
        tx, ty = rng.integers(T * 7 // 8, T + 1, 2)
        x = (np.cumsum(rng.standard_normal((tx, D)), 0) * 0.3).astype(np.float32)
        X[i, :tx] = x
        idx = np.minimum(np.arange(ty) * tx // ty, tx - 1)
        Y[i, :ty] = x[idx] + 0.05 * rng.standard_normal((ty, D)).astype(np.float32)
    Xa, Ya = DTWAligner(dist=melcd, radius=1).transform((X, Y))
    return np.concatenate((Xa, Ya), axis=-1).reshape(-1, 2 * D)


def vc_matrix(seed=1, N=200000, D=72, K=64):
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((K, D)) * 2.0
    lab = rng.integers(0, K, N)
    X = centres[lab] + rng.standard_normal((N, D)) * rng.uniform(0.3, 1.2, (K, D))[lab]
    X[:, 0] += 30.0  # c0-like dimension
    return X.astype(np.float32)


def run(name, X, K, iters, do_sklearn):
    import torch
    from sklearn.mixture import GaussianMixture as Sk
    from sklearn.utils import check_random_state

    from nnmnkwii_b200.baseline import gmm as G
    N, D = X.shape
    flop = 2.0 * N * K * D * (D + 1)
    est = G.GaussianMixture(n_components=K, random_state=0)
    t0 = time.perf_counter()
    resp = est._initial_resp(N, lambda: X.astype(np.float64), check_random_state(0))
    t_init = time.perf_counter() - t0
    Xd = torch.from_numpy(X).cuda()
    st = G._EmState(Xd, K, est.reg_covar)
    st.put("resp", resp)
    st.mstep(0)
    st.factor(True)
    st.check_status()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    e_ms, m_ms = [], []
    for _ in range(iters + 1):
        ev[0].record()
        st.estep()
        ev[1].record()
        st.mstep(1)
        st.factor(True)
        ev[2].record()
        ev[2].synchronize()
        e_ms.append(ev[0].elapsed_time(ev[1]))
        m_ms.append(ev[1].elapsed_time(ev[2]))
    st.check_status()
    e_ms, m_ms = e_ms[1:], m_ms[1:]  # the first iteration includes module load / attribute setup
    it_ms = float(np.median(np.add(e_ms, m_ms)))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fit = G.GaussianMixture(n_components=K, random_state=0, max_iter=100).fit(X)
        t_fit = time.perf_counter() - t0
        sk_s = None
        if do_sklearn:
            sk = Sk(n_components=K, max_iter=2, tol=0.0, weights_init=fit.weights_, means_init=fit.means_,
                    precisions_init=fit.precisions_)
            X64 = X.astype(np.float64)
            t0 = time.perf_counter()
            sk.fit(X64)
            sk_s = (time.perf_counter() - t0) / 2.0
    rec = {
        "workload": name, "N": int(N), "D": int(D), "K": int(K),
        "em_iter_ms_median": round(it_ms, 4),
        "estep_ms_median": round(float(np.median(e_ms)), 4),
        "mstep_factor_ms_median": round(float(np.median(m_ms)), 4),
        "fp64_flop_per_iter": flop,
        "achieved_fp64_tflops": round(flop / (it_ms * 1e-3) / 1e12, 3),
        "share_of_fp64_peak_34T": round(flop / (it_ms * 1e-3) / PEAK_FP64, 4),
        "share_of_fp64_tc_peak_67T": round(flop / (it_ms * 1e-3) / PEAK_FP64_TC, 4),
        "host_init_kmeans_s": round(t_init, 3),
        "device_fit_wall_s": round(t_fit, 3), "device_fit_n_iter": int(fit.n_iter_),
        "sklearn_s_per_iter_2iter_timing": None if sk_s is None else round(sk_s, 3),
        "host_cpus": os.cpu_count(),
    }
    print(json.dumps(rec), flush=True)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--workloads", default="aligner,vc")
    ap.add_argument("--no-sklearn", action="store_true")
    args = ap.parse_args()
    import torch
    torch.cuda.set_device(0)
    name, plim = card()
    print(json.dumps({"card": name, "power_limit": plim}), flush=True)
    for w in args.workloads.split(","):
        if w == "aligner":
            run("aligner_configs3", aligner_matrix(), 16, args.iters, not args.no_sklearn)
        elif w == "vc":
            run("vc_72x64", vc_matrix(), 64, args.iters, not args.no_sklearn)
        else:
            raise SystemExit("unknown workload %r" % w)


if __name__ == "__main__":
    main()
