"""GMM-based voice conversion -- drop-in for ``nnmnkwii.baseline.gmm`` (baseline/gmm.py:47-247).

SURVEY.md section 8f row 1: the in-repo caller that turns a joint source/target GMM and a source
utterance into the per-frame means ``E`` (Eq. 22) and diagonal variances ``D`` (Eq. 23) that
``paramgen.mlpg`` consumes.  The reference walks the frames in Python (one ``np.linalg.solve`` per
frame); here the mixture posteriors, the per-frame affine maps and the variances are evaluated for a
whole utterance -- or a whole batch of utterances -- on the GPU in float64 and handed to the MLPG
kernels without leaving the device.

``GaussianMixture`` fits the joint GMM itself: scikit-learn's estimator with its EM iterations run by the
float64 kernels of csrc/nnk_gmm_em.cu (C ABI ``nnk_gmm_em_*``).

The per-mixture matrices ``A[m] = covarYX[m] covarXX[m]^-1`` are formed once (the reference re-solves
per frame, gmm.py:113-115, 231-233).  Posteriors, arg-max mixture, affine map and variances run in the
float64 kernels of csrc/nnk_gmm.cu (C ABI ``nnk_gmm_logprob`` / ``nnk_gmm_map``): no (frames, mixtures,
dim) temporaries, ``E`` and ``D`` are written directly in the layout the MLPG kernels read.
"""
import ctypes
import math

import numpy as np
from scipy import linalg
from sklearn.mixture import GaussianMixture as _SkGaussianMixture

from ..paramgen import mlpg_batch, mlpg_gv_batch, mlpg_ms_batch


def _compute_precision_cholesky_full(covariances):
    """Upper factors U with U U^T = covariance^-1, as scikit-learn stores them (gmm.py:8-41)."""
    n_components, n_features, _ = covariances.shape
    out = np.empty((n_components, n_features, n_features))
    for k, cov in enumerate(covariances):
        try:
            c = linalg.cholesky(cov, lower=True)
        except linalg.LinAlgError:
            raise ValueError(
                "Fitting the mixture model failed because some components have ill-defined empirical "
                "covariance (for instance caused by singleton or collapsed samples). Try to decrease the "
                "number of components, or increase reg_covar.")
        out[k] = linalg.solve_triangular(c, np.eye(n_features), lower=True).T
    return out


class MLPGBase(object):
    """Frame-wise GMM mapping ``E[p(y | x)]`` (baseline/gmm.py:47-121)."""

    def __init__(self, gmm, swap=False, diff=False):
        assert gmm.covariance_type == "full"
        D = gmm.means_.shape[1] // 2  # static + delta dim
        self.num_mixtures = gmm.means_.shape[0]
        self.weights = gmm.weights_
        self.src_means = gmm.means_[:, :D]
        self.tgt_means = gmm.means_[:, D:]
        self.covarXX = gmm.covariances_[:, :D, :D]
        self.covarXY = gmm.covariances_[:, :D, D:]
        self.covarYX = gmm.covariances_[:, D:, :D]
        self.covarYY = gmm.covariances_[:, D:, D:]
        if diff:  # GMM -> DIFFGMM (gmm.py:63-67)
            self.tgt_means = self.tgt_means - self.src_means
            self.covarYY = self.covarXX + self.covarYY - self.covarXY - self.covarYX
            self.covarXY = self.covarXY - self.covarXX
            self.covarYX = self.covarXY.transpose(0, 2, 1)
        if swap:  # (gmm.py:70-73)
            self.tgt_means, self.src_means = self.src_means, self.tgt_means
            self.covarYY, self.covarXX = self.covarXX, self.covarYY
            self.covarYX, self.covarXY = self.covarXY, self.covarYX
        self._prec_chol = _compute_precision_cholesky_full(self.covarXX)
        self._dev = None

    # ---- device-side constants -------------------------------------------------------------------
    def _constants(self):
        import torch

        from .. import _device as dev
        dev.require_cuda()
        device = dev.cuda_device()
        if self._dev is not None and self._dev["device"] == device:
            return self._dev

        def t(a):
            return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(device)
        A = np.stack([np.linalg.solve(self.covarXX[m].T, self.covarYX[m].T).T for m in range(self.num_mixtures)])
        dim = self.src_means.shape[1]
        log_det = np.sum(np.log(np.diagonal(self._prec_chol, axis1=1, axis2=2)), axis=1)
        Dm = self._diag_variances()
        from .. import _lib
        tabs = {
            "src_means": t(self.src_means), "tgt_means": t(self.tgt_means), "prec_chol": t(self._prec_chol),
            "log_const": t(log_det + np.log(self.weights) - 0.5 * dim * np.log(2.0 * np.pi)),
            "A_t": t(A.transpose(0, 2, 1)), "Dm": t(Dm),
        }
        g = _lib.NnkGmm()
        for k, v in tabs.items():
            setattr(g, k, v.data_ptr())
        g.M, g.D = self.num_mixtures, dim
        self._dev = {"device": device, "tabs": tabs, "gmm": g}
        return self._dev

    def _diag_variances(self):
        """Eq. (23) with diagonal covariances (gmm.py:239-244), (M, D)."""
        return np.stack([np.diag(self.covarYY[m]) - np.diag(self.covarYX[m]) / np.diag(self.covarXX[m]) * np.diag(self.covarXY[m])
                         for m in range(self.num_mixtures)])

    def _to_device(self, src):
        import torch
        c = self._constants()
        return torch.from_numpy(np.ascontiguousarray(src, dtype=np.float64)).to(c["device"]), c

    def _weighted_log_prob(self, x, c):
        """log w_m + log N(x_t | mu_m, Sigma_xx,m) for every frame and mixture, (T, M) (Eq. 9 before
        normalisation; the reference: sklearn predict_proba per frame, gmm.py:116-118)."""
        import torch

        from .. import _device as dev
        from .. import _lib
        T = x.shape[0]
        lp = torch.empty((T, self.num_mixtures), dtype=torch.float64, device=x.device)
        _lib.check(_lib.lib.nnk_gmm_logprob(ctypes.byref(c["gmm"]), x.data_ptr(), x.stride(0), T, lp.data_ptr(),
                                            dev.current_stream_ptr(x.device)), "nnk_gmm_logprob")
        return lp

    def _map(self, x, c, mode, want_var=False, lp=None):
        """mode 0: (E, D, mix) of the arg-max mixture sequence (Eq. 37, 22, 23); mode 1: posterior mean (Eq. 13).
        ``lp``: the ``_weighted_log_prob`` of ``x`` if the caller already has it."""
        import torch

        from .. import _device as dev
        from .. import _lib
        T, D = x.shape
        if lp is None:
            lp = self._weighted_log_prob(x, c)
        E = torch.empty((T, D), dtype=torch.float64, device=x.device)
        Dv = torch.empty((T, D), dtype=torch.float64, device=x.device) if want_var else None
        _lib.check(_lib.lib.nnk_gmm_map(ctypes.byref(c["gmm"]), x.data_ptr(), x.stride(0), T, lp.data_ptr(), mode, E.data_ptr(),
                                        Dv.data_ptr() if want_var else None, None, dev.current_stream_ptr(x.device)),
                   "nnk_gmm_map")
        return E, Dv

    def transform(self, src):
        src = np.asarray(src)
        if src.ndim == 2:
            tgt = np.zeros_like(src)
            if len(src):
                tgt[:] = self._transform_frames(src)  # zeros_like keeps the dtype of src (gmm.py:89-93)
            return tgt
        return self._transform_frames(src[None])[0]

    def _transform_frame(self, src):
        """``E[p(y | x)]`` of one frame (gmm.py:97-121)."""
        return self._transform_frames(np.asarray(src)[None])[0]

    def _transform_frames(self, src):
        xa, c = self._to_device(src)
        if xa.shape[0] == 0:
            return xa.cpu().numpy()
        E, _ = self._map(xa.contiguous(), c, 1)  # Eq. (9), (11), (13) in one pass per frame tile
        return E.cpu().numpy()


class MLPG(MLPGBase):
    """Maximum likelihood parameter generation for GMM-based voice conversion (baseline/gmm.py:124-247).

    Args:
        gmm (sklearn.mixture.GaussianMixture): joint GMM of source and target features.
        windows (list): window triples, see :func:`nnmnkwii_b200.paramgen.mlpg`.
        swap (bool): if True source -> target, otherwise target -> source.
        diff (bool): convert GMM -> DIFFGMM if True.
        gv (tuple): additive: ``(gv_mean, gv_var)`` of the target's static features, each of length
            ``static_dim`` (e.g. :func:`nnmnkwii_b200.paramgen.gv_statistics` of the training targets).
            When given, :meth:`transform` and :meth:`transform_batch` generate with
            :func:`nnmnkwii_b200.paramgen.mlpg_gv_batch` (Toda, Black & Tokuda 2007, Sec. IV) instead of
            plain MLPG.  Not defined for ``diff=True`` (``ValueError``), and not applied on the
            posterior-mean path (source features of ``static_dim`` columns), which runs no MLPG.
        ms (tuple): additive: ``(ms_mean, ms_var)``, statistics of the log modulation spectrum of the target's
            static features, each ``(n // 2 + 1, static_dim)`` (e.g.
            :func:`nnmnkwii_b200.postfilters.modspec_statistics` of natural static trajectories).  When given,
            :meth:`transform` and :meth:`transform_batch` generate with
            :func:`nnmnkwii_b200.paramgen.mlpg_ms_batch` instead of plain MLPG.  ``ValueError`` together with
            ``gv``, with ``diff=True`` and for :meth:`transform_em`; not applied on the posterior-mean path.
        ms_segment (int): additive: the segment length ``L`` of a segment-level ``ms``
            (``mlpg_ms_batch(..., segment=L)``, statistics from ``modspec_statistics(..., segment=L)`` with
            ``n`` 32 .. 512), for utterances of any length.  ``ValueError`` without ``ms``.
    """

    def __init__(self, gmm, windows=None, swap=False, diff=False, gv=None, ms=None, ms_segment=None):
        super(MLPG, self).__init__(gmm, swap, diff)
        if windows is None:
            windows = [(0, 0, np.array([1.0])), (1, 1, np.array([-0.5, 0.0, 0.5]))]
        self.windows = windows
        self.static_dim = gmm.means_.shape[-1] // 2 // len(windows)
        self.gv = None
        if gv is not None:
            if diff:
                raise ValueError("gv is not defined for difference features (diff=True)")
            gv_mean, gv_var = (np.asarray(a, dtype=np.float64).ravel() for a in gv)
            from ..paramgen import StreamLayout, _gv_args
            _gv_args(gv_mean, gv_var, StreamLayout.single(self.static_dim * len(windows), len(windows)), 0, 1.0, None)
            self.gv = (gv_mean, gv_var)
        self.ms = None
        self.ms_segment = None
        if ms_segment is not None and ms is None:
            raise ValueError("ms_segment needs ms (segment-level MS statistics)")
        if ms is not None:
            if gv is not None:
                raise ValueError("ms and gv cannot be combined")
            if diff:
                raise ValueError("ms is not defined for difference features (diff=True)")
            from ..paramgen import StreamLayout, _ms_args
            ms_mean, ms_var = _ms_args(ms[0], ms[1], StreamLayout.single(self.static_dim * len(windows), len(windows)),
                                       0, 1.0, None, ms_segment)[:2]
            self.ms = (ms_mean, ms_var)
            self.ms_segment = None if ms_segment is None else int(ms_segment)

    def _generate(self, E, Dv, lengths):
        if self.ms is not None:
            return mlpg_ms_batch(E, Dv, self.windows, self.ms[0], self.ms[1], lengths=lengths,
                                 segment=self.ms_segment)
        if self.gv is None:
            return mlpg_batch(E, Dv, self.windows, lengths=lengths)
        return mlpg_gv_batch(E, Dv, self.windows, self.gv[0], self.gv[1], lengths=lengths)

    def _means_vars(self, x, c):
        """E (Eq. 22) and D (Eq. 23) of the sub-optimum mixture sequence (Eq. 37), on the device."""
        return self._map(x.contiguous(), c, 0, want_var=True)

    def transform(self, src):
        """Source feature sequence ``(T, D)`` -> converted static features ``(T, static_dim)``."""
        src = np.asarray(src)
        T, feature_dim = src.shape[0], src.shape[1]
        if feature_dim == self.static_dim:
            return super(MLPG, self).transform(src)
        x, c = self._to_device(src)
        E, Dv = self._means_vars(x, c)
        return self._generate(E, Dv, [T]).cpu().numpy()

    def transform_batch(self, srcs):
        """Additive: convert a list of utterances in one pass (one posterior / mapping evaluation and
        ONE batched MLPG launch for all of them).  Returns a list of ``(T_i, static_dim)`` arrays."""
        import torch
        lens = [len(s) for s in srcs]
        if not lens:
            return []
        flat = np.concatenate([np.asarray(s) for s in srcs], axis=0)
        if flat.shape[1] == self.static_dim:
            y = MLPGBase._transform_frames(self, flat)
        else:
            x, c = self._to_device(flat)
            E, Dv = self._means_vars(x, c)
            y = self._generate(E, Dv, lens).cpu().numpy()
        del torch
        off = np.concatenate([[0], np.cumsum(lens)])
        return [y[off[i]:off[i + 1]] for i in range(len(lens))]

    def transform_em(self, src, n_iter=5, return_log_likelihood=False):
        """Additive: source features ``(T, D)`` -> converted static features ``(T, static_dim)`` float64, by
        maximum-likelihood conversion over all mixture sequences (Toda, Black & Tokuda 2007, Sec. III).

        The trajectory ``c`` maximises ``L(c) = sum_t log sum_m exp(lp[t, m] + log N(Y_t; E_{m,t}, diag D_m))``
        with ``Y = W c`` its static + dynamic sequence (windows never cross the utterance; on the first and last
        ``H = max(l, u)`` frames, and on every frame of a window set with ``H = 0``, only the static columns count,
        as :func:`~nnmnkwii_b200.paramgen.mlpg` gives the dynamic windows zero precision there), ``E_{m,t}`` the
        Eq. 22 mean, ``D_m`` the diagonal Eq. 23 variances :meth:`transform` uses and
        ``lp[t, m] = log w_m + log N(x_t; mu_m, Sigma_xx,m)``.  EM from ``c_0 = transform(src)``: the E-step
        gives the mixture posteriors ``gamma[t, m]`` of the current trajectory, the M-step is one MLPG solve with
        precisions ``P_t = sum_m gamma[t, m] / D_m`` and means ``(sum_m gamma[t, m] E_{m,t} / D_m) / P_t``, so
        ``L`` never decreases.  This is an exact EM for the diagonal-``D_m`` model of :meth:`transform`; the
        paper's posterior uses the full conditional covariance instead.  E-step, M-step and the objective run
        on the GPU in float64 with one host synchronisation, when the result comes back.

        Args:
            src: ``(T, D)`` source features with static and dynamic columns.
            n_iter (int): EM iterations; 0 returns exactly what :meth:`transform` returns.
            return_log_likelihood (bool): also return ``L`` at ``c_0 .. c_{n_iter}``, ``(n_iter + 1,)`` float64.

        Raises ``ValueError`` when ``gv`` is set, when ``src`` has ``static_dim`` columns (the posterior-mean
        path runs no MLPG), for ``n_iter < 0`` or a ``D_m`` entry that is not positive and finite, and
        ``NotImplementedError`` for ``D > 96``; all before anything is launched."""
        out = self.transform_em_batch([src], n_iter=n_iter, return_log_likelihood=return_log_likelihood)
        if return_log_likelihood:
            return out[0][0], out[1][0]
        return out[0]

    def transform_em_batch(self, srcs, n_iter=5, return_log_likelihood=False):
        """Additive: :meth:`transform_em` of a list of utterances in one flat batch on the device (one E-step
        launch and one batched MLPG solve per iteration for all of them).  Returns the list of
        ``(T_i, static_dim)`` arrays, and with ``return_log_likelihood`` also an ``(n_utt, n_iter + 1)`` array."""
        import torch

        from .. import _device as dev
        from .. import _lib
        from ..paramgen import StreamLayout, _utterance_table
        srcs = [np.asarray(s) for s in srcs]
        n_iter = self._check_em(srcs, n_iter)
        lens = [len(s) for s in srcs]
        nw, S = len(self.windows), self.static_dim
        if not lens or not sum(lens):
            ys = [np.zeros((n, S)) for n in lens]
            return (ys, np.zeros((len(lens), n_iter + 1))) if return_log_likelihood else ys
        x, c = self._to_device(np.concatenate(srcs, axis=0))
        T, D = x.shape
        device = x.device
        em = self._em_constants(c)

        def up(a):  # asynchronous upload: nothing below waits for the device until the results come back
            return torch.from_numpy(np.ascontiguousarray(a)).pin_memory().to(device, non_blocking=True)
        off, ulens, order, max_T, n_utt = _utterance_table(lens, None, T)
        layout = StreamLayout.single(D, nw)
        win = _lib.make_windows(self.windows)
        offsets, order_d, chains = up(off), up(order), dev.chains_on_device(layout.chains, device)
        status = torch.zeros(1, dtype=torch.int64, device=device)
        tiles = -(-ulens // _lib.NNK_GMM_TRAJ_TILE)
        tile_off = np.concatenate([[0], np.cumsum(tiles)]).astype(np.int32)
        tables = up(np.concatenate([off.astype(np.int32), tile_off]))
        n_tiles = int(tile_off[-1])

        def solve(E, V):  # the kernels and arguments of mlpg_batch(E, V, windows, lengths=lens)
            y = torch.zeros((T, S), dtype=torch.float64, device=device)
            dev.run_mlpg("fwd", means=E, variances=V, rhs=None, out=y, offsets=offsets, lengths=None, order=order_d,
                         chains=chains, n_chain=layout.n_chain, max_T=max_T, windows_c=win, in_ld=D, var_ld=D,
                         go_ld=0, out_ld=S, dtype_code=_lib.NNK_F64, go_f64=0, n_utt=n_utt, device=device,
                         check=False, status=status)
            return y

        lp = self._weighted_log_prob(x, c)
        E, V = self._map(x, c, 0, want_var=True, lp=lp)
        y = solve(E, V)
        ll = torch.zeros((n_iter + 1, max(n_tiles, 1)), dtype=torch.float64, device=device)
        a = _lib.NnkGmmTrajArgs()
        a.x, a.x_ld, a.lp, a.T, a.n_utt = x.data_ptr(), x.stride(0), lp.data_ptr(), T, n_utt
        a.utt_off, a.tile_off, a.n_tiles = tables.data_ptr(), tables.data_ptr() + 4 * (n_utt + 1), n_tiles
        a.static_dim, a.win = S, win
        a.inv_Dm, a.log_norm = em["inv_Dm"].data_ptr(), em["log_norm"].data_ptr()
        E_bar = torch.empty((T, D), dtype=torch.float64, device=device)
        V_bar = torch.empty((T, D), dtype=torch.float64, device=device)
        a.E_bar, a.V = E_bar.data_ptr(), V_bar.data_ptr()
        for k in range(n_iter + (1 if return_log_likelihood else 0)):
            a.c, a.c_ld = y.data_ptr(), y.stride(0)
            a.mode = _lib.NNK_GMM_TRAJ_EM if k < n_iter else _lib.NNK_GMM_TRAJ_OBJECTIVE
            a.ll_part = ll[k].data_ptr() if return_log_likelihood else None
            _lib.check(_lib.lib.nnk_gmm_traj_em(ctypes.byref(c["gmm"]), ctypes.byref(a), dev.current_stream_ptr(device)),
                       "nnk_gmm_traj_em")
            if k < n_iter:
                y = solve(E_bar, V_bar)
        dev.raise_if_failed(status)
        y = y.cpu().numpy()
        bounds = np.concatenate([[0], np.cumsum(lens)])
        ys = [y[bounds[i]:bounds[i + 1]] for i in range(len(lens))]
        if not return_log_likelihood:
            return ys
        parts = ll.cpu().numpy()
        L = np.array([[math.fsum(parts[k, tile_off[u]:tile_off[u + 1]]) for k in range(n_iter + 1)]
                      for u in range(n_utt)])
        return ys, L

    def _check_em(self, srcs, n_iter):
        """The arguments :meth:`transform_em_batch` refuses, before anything is launched; returns ``n_iter``."""
        if self.gv is not None:
            raise ValueError("transform_em does not combine EM with global variance (gv is set)")
        if self.ms is not None:
            raise ValueError("transform_em does not combine EM with the modulation spectrum (ms is set)")
        D = self.src_means.shape[1]
        for s in srcs:
            if s.ndim != 2:
                raise ValueError("transform_em expects (T, D) utterances (got shape %s)" % (s.shape,))
            if s.shape[1] == self.static_dim:
                raise ValueError("transform_em needs static and dynamic source features: the posterior-mean path "
                                 "(%d columns) runs no MLPG" % s.shape[1])
            if s.shape[1] != D:
                raise ValueError("source features have %d columns, the GMM %d" % (s.shape[1], D))
        if isinstance(n_iter, (bool, np.bool_)) or int(n_iter) != n_iter or n_iter < 0:
            raise ValueError("n_iter must be a non-negative integer (got %r)" % (n_iter,))
        Dm = self._diag_variances()
        if not np.all(np.isfinite(Dm) & (Dm > 0)):
            raise ValueError("transform_em needs positive, finite Eq. (23) variances D_m")
        if D > 96:
            raise NotImplementedError("feature dimension > 96 is not supported by the GMM kernels")
        return int(n_iter)

    def _em_constants(self, c):
        """1 / D_m and -1/2 (sum_d log D_m,d + n log 2 pi) over all n = D columns and over the static ones (the
        columns an utterance's edge frames keep, see include/nnk_b200.h) on the device, cached with the
        other tables."""
        if "em" not in c:
            import torch
            Dm = self._diag_variances()
            inv = np.ascontiguousarray(1.0 / Dm)
            S = self.static_dim
            log_norm = -0.5 * np.stack([np.sum(np.log(Dm), axis=1) + Dm.shape[1] * np.log(2.0 * np.pi),
                                        np.sum(np.log(Dm[:, :S]), axis=1) + S * np.log(2.0 * np.pi)], axis=1)
            c["em"] = {k: torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64)).to(c["device"])
                       for k, v in (("inv_Dm", inv), ("log_norm", log_norm))}
        return c["em"]


_EM_MAX_FEATURES = 128
_EM_MAX_COMPONENTS = 128
_ILL_DEFINED = ("Fitting the mixture model failed because some components have ill-defined empirical covariance "
                "(for instance caused by singleton or collapsed samples). Try to decrease the number of components, "
                "increase reg_covar, or scale the input data.")


class _EmState(object):
    """Device buffers of one fit: the frames, the responsibilities, the parameters, the workspace of
    csrc/nnk_gmm_em.cu and the filled ``nnk_gmm_em_args_t``.  Each step runs on the current stream at the
    time of the call.  The buffers belong to the stream current at construction, so a step on another
    stream must be ordered after that stream's work, and the object must outlive the steps it enqueued
    (within ``fit_predict`` both hold: one stream, synchronising steps)."""

    def __init__(self, X, K, reg_covar):
        import torch

        from .. import _device as dev
        from .. import _lib
        self.X, self.device = X, X.device
        N, D = X.shape
        f64 = dict(dtype=torch.float64, device=X.device)
        self.resp = torch.empty((N, K), **f64)
        self.weights = torch.empty(K, **f64)
        self.means = torch.empty((K, D), **f64)
        self.covariances = torch.empty((K, D, D), **f64)
        self.prec_chol = torch.empty((K, D, D), **f64)
        self.lower_bound = torch.zeros(1, **f64)
        self.status = torch.zeros(1, dtype=torch.int32, device=X.device)
        nbytes = _lib.lib.nnk_gmm_em_workspace_bytes(N, D, K)
        self.ws = dev.workspace(X.device, nbytes)
        a = _lib.NnkGmmEmArgs()
        a.X, a.N, a.x_ld, a.dtype, a.D, a.K = X.data_ptr(), N, X.stride(0), dev.torch_dtype_code(X.dtype), D, K
        a.reg_covar = float(reg_covar)
        for name in ("resp", "weights", "means", "covariances", "prec_chol", "lower_bound", "status"):
            setattr(a, name, getattr(self, name).data_ptr())
        a.workspace, a.workspace_bytes = self.ws.data_ptr(), self.ws.numel()
        self.args = a

    def _call(self, name):
        from .. import _device as dev
        from .. import _lib
        # the caller's current stream at each step, like every other launcher
        _lib.check(getattr(_lib.lib, name)(ctypes.byref(self.args), dev.current_stream_ptr(self.X.device)), name)

    def estep(self):
        self._call("nnk_gmm_em_estep")

    def mstep(self, weight_norm):
        self.args.weight_norm = weight_norm
        self._call("nnk_gmm_em_mstep")

    def factor(self, factor):
        self.args.factor = int(factor)
        self._call("nnk_gmm_em_factor")

    def put(self, name, array):
        import torch
        getattr(self, name).copy_(torch.from_numpy(np.ascontiguousarray(array, dtype=np.float64)))

    def check_status(self):
        """Synchronises: raises sklearn's ValueError if a Cholesky pivot was not positive."""
        if int(self.status.item()):
            raise ValueError(_ILL_DEFINED)


def _as_frames(X):
    """(N, D) frames for the device: numpy / array-likes are validated like sklearn and uploaded; CUDA
    tensors stay where they are.  Returns (device tensor, host float64 array or None)."""
    import torch

    from .. import _device as dev
    from sklearn.utils import check_array
    dev.require_cuda()
    if isinstance(X, torch.Tensor) and X.is_cuda:
        if X.ndim != 2:
            raise ValueError("Expected 2D array, got %dD tensor instead" % X.ndim)
        if X.dtype not in (torch.float32, torch.float64):
            X = X.to(torch.float64)
        if X.shape[0] < 2:
            raise ValueError("Found array with %d sample(s) (shape=%s) while a minimum of 2 is required by "
                             "GaussianMixture." % (X.shape[0], tuple(X.shape)))
        if not bool(torch.isfinite(X).all()):
            raise ValueError("Input X contains NaN or infinity.")
        if X.shape[1] == 0 or X.stride(1) != 1 or X.stride(0) < X.shape[1]:
            X = X.contiguous()
        return X, None
    if isinstance(X, torch.Tensor):
        X = X.numpy()
    Xh = check_array(X, dtype=[np.float64, np.float32], ensure_min_samples=2, estimator="GaussianMixture")
    return dev.to_device(Xh), Xh


def _host_f64(t):
    return t.detach().cpu().numpy().astype(np.float64, copy=True)


_KM_MAX_FEATURES = 128
_KM_MAX_CLUSTERS = 128


def _check_kmeans_sizes(Xd, K):
    """The limits of csrc/nnk_kmeans.cu, raised before anything is launched."""
    import torch
    N, D = Xd.shape
    if not 1 <= D <= _KM_MAX_FEATURES:
        raise ValueError("k-means on the GPU supports 1 to %d features (got %d)" % (_KM_MAX_FEATURES, D))
    if not 1 <= K <= _KM_MAX_CLUSTERS:
        raise ValueError("k-means on the GPU supports 1 to %d clusters (got %d)" % (_KM_MAX_CLUSTERS, K))
    if N < K:
        raise ValueError("n_samples=%d should be >= n_clusters=%d." % (N, K))
    if Xd.dtype not in (torch.float32, torch.float64) or Xd.stride(1) != 1 or Xd.stride(0) < D:
        raise ValueError("k-means on the GPU reads float32 / float64 rows with unit column stride")


def _kmeans_plusplus_draws(N, K, random_state):
    """The RandomState calls of sklearn's ``_kmeans_plusplus`` (unit sample weights), in its order: the first
    centre, then ``n_local_trials`` uniforms per later centre.  Returns (first, (K - 1, trials) array)."""
    trials = 2 + int(np.log(K))
    sample_weight = np.ones(N, dtype=np.float64)
    first = int(random_state.choice(N, p=sample_weight / sample_weight.sum()))
    u = np.empty((K - 1, trials), dtype=np.float64)
    for c in range(1, K):
        u[c - 1] = random_state.uniform(size=trials)
    return first, u


class _KMeansState(object):
    """Device buffers of one k-means run over the frames ``X`` (csrc/nnk_kmeans.cu) and the filled
    ``nnk_kmeans_args_t``.  ``centre``: KMeans reads the rows minus their mean, kmeans_plusplus the raw rows.
    Steps run on the current stream at the time of the call; the buffers belong to the stream current at
    construction, with the same ordering and lifetime rules as ``_EmState``."""

    def __init__(self, X, K, centre):
        import torch

        from .. import _device as dev
        from .. import _lib
        _check_kmeans_sizes(X, K)
        self.X, self.K = X, K
        N, D = X.shape
        f64 = dict(dtype=torch.float64, device=X.device)
        self.labels = torch.full((N,), -1, dtype=torch.int32, device=X.device)
        self.centers = torch.zeros((K, D), **f64)
        self.sums = torch.zeros((K, D), **f64)
        self.weights = torch.zeros(K, **f64)
        self.indices = torch.zeros(K, dtype=torch.int64, device=X.device)
        self.mean = torch.zeros(D, **f64)
        self.out_centers = torch.zeros((K, D), **f64)
        self.status = torch.zeros(_lib.NNK_KM_STATUS_LEN, **f64)
        self.dist = None
        self.rand = None
        self.ws = dev.workspace(X.device, _lib.lib.nnk_kmeans_workspace_bytes(N, D, K))
        a = _lib.NnkKmeansArgs()
        a.X, a.N, a.x_ld, a.dtype, a.D, a.K = X.data_ptr(), N, X.stride(0), dev.torch_dtype_code(X.dtype), D, K
        a.centre = int(bool(centre))
        for name in ("centers", "sums", "weights", "labels", "indices", "mean", "out_centers", "status"):
            setattr(a, name, getattr(self, name).data_ptr())
        a.workspace, a.workspace_bytes = self.ws.data_ptr(), self.ws.numel()
        self.args = a

    def _call(self, name):
        from .. import _device as dev
        from .. import _lib
        # the caller's current stream at each step, like every other launcher
        _lib.check(getattr(_lib.lib, name)(ctypes.byref(self.args), dev.current_stream_ptr(self.X.device)), name)

    def read_status(self):
        """Synchronises: the small status record of the last call."""
        return self.status.cpu().numpy()

    def prepare(self):
        self._call("nnk_kmeans_prepare")

    def seed(self, first, u):
        import torch
        self.rand = torch.from_numpy(np.ascontiguousarray(u, dtype=np.float64)).to(self.X.device)
        self.args.first = int(first)
        self.args.rand = self.rand.data_ptr() if self.rand.numel() else None
        self._call("nnk_kmeans_seed")

    def lloyd(self, update):
        self.args.update = int(bool(update))
        self._call("nnk_kmeans_lloyd")

    def relocate_empty_clusters(self):
        """sklearn's ``_relocate_empty_clusters_dense`` on the sums and weights of the last Lloyd step.  The
        distances come from the device; the choice of samples is numpy's own ``argpartition``, because the
        order of its introselect among the farthest samples is not something a kernel can restate.  Only the
        chosen rows are downloaded.  Rare: k-means++ seeds seldom leave a cluster empty."""
        import torch
        if self.dist is None:
            self.dist = torch.empty(self.X.shape[0], dtype=torch.float64, device=self.X.device)
            self.args.dist = self.dist.data_ptr()
        self._call("nnk_kmeans_relocate_dist")
        distances = self.dist.cpu().numpy()
        weights = self.weights.cpu().numpy()
        empty = np.where(np.equal(weights, 0))[0]
        n_empty = empty.shape[0]
        far = np.argpartition(distances, -n_empty)[:-n_empty - 1:-1]
        if np.max(distances) == 0:
            return
        sums = self.sums.cpu().numpy()
        far_t = torch.from_numpy(far.astype(np.int64)).to(self.X.device)
        rows = self.X[far_t].to(torch.float64).cpu().numpy() - self.mean.cpu().numpy()
        labels = self.labels[far_t].cpu().numpy()
        for idx in range(n_empty):
            new, old, weight = empty[idx], labels[idx], 1.0
            sums[old] -= rows[idx] * weight
            sums[new] = rows[idx] * weight
            weights[new] = weight
            weights[old] -= weight
        self.sums.copy_(torch.from_numpy(sums))
        self.weights.copy_(torch.from_numpy(weights))

    def average(self):
        self._call("nnk_kmeans_average")

    def inertia(self):
        self._call("nnk_kmeans_inertia")


def _device_kmeans_plusplus(Xd, K, random_state):
    """sklearn's public ``kmeans_plusplus(X, K, random_state=...)`` on the raw rows of the device frames ``Xd``
    (no centring, as that function does not centre): returns (centers (K, D) float64, indices (K,) int64),
    both CUDA tensors.  ``random_state`` is consumed exactly as scikit-learn consumes it."""
    from sklearn.utils import check_random_state
    _check_kmeans_sizes(Xd, K)
    first, u = _kmeans_plusplus_draws(Xd.shape[0], K, check_random_state(random_state))
    st = _KMeansState(Xd, K, centre=False)
    st.prepare()
    st.seed(first, u)
    return st.centers, st.indices


def _device_kmeans(Xd, K, random_state=None, init=None, max_iter=300, tol=1e-4):
    """sklearn's ``KMeans(n_clusters=K, n_init=1, init=init or "k-means++", max_iter, tol, random_state).fit``
    (Lloyd) on the device frames ``Xd``.  Returns (labels (N,) int64 CUDA tensor, centers (K, D) float64 CUDA
    tensor, inertia, n_iter).  One small status record is read back per iteration."""
    import warnings

    import torch
    from sklearn.exceptions import ConvergenceWarning
    from sklearn.utils import check_random_state

    from .. import _lib
    _check_kmeans_sizes(Xd, K)
    if int(max_iter) < 1:
        raise ValueError("max_iter must be >= 1 (got %r)" % (max_iter,))
    if init is not None:
        init = np.array(init, dtype=np.float64, copy=True)
        if init.shape != (K, Xd.shape[1]):
            raise ValueError("init should be of shape %s, got %s" % ((K, Xd.shape[1]), init.shape))
    st = _KMeansState(Xd, K, centre=True)
    st.prepare()
    if init is None:
        first, u = _kmeans_plusplus_draws(Xd.shape[0], K, check_random_state(random_state))
        st.seed(first, u)
        s = st.read_status()
    else:
        s = st.read_status()
        init -= st.mean.cpu().numpy()
        st.centers.copy_(torch.from_numpy(init))
    tol_abs = 0.0 if tol == 0 else float(s[_lib.NNK_KM_VAR_MEAN]) * tol
    strict = False
    for i in range(int(max_iter)):
        st.lloyd(True)
        s = st.read_status()
        if s[_lib.NNK_KM_EMPTY] > 0:
            st.relocate_empty_clusters()
            st.average()
            s = st.read_status()
        if s[_lib.NNK_KM_CHANGED] == 0:
            strict = True
            break
        if s[_lib.NNK_KM_SHIFT] <= tol_abs:
            break
    if not strict:
        st.lloyd(False)  # labels that match the final centres
    st.inertia()
    s = st.read_status()
    distinct = int(s[_lib.NNK_KM_DISTINCT])
    if distinct < K:
        warnings.warn("Number of distinct clusters ({}) found smaller than n_clusters ({}). Possibly due to "
                      "duplicate points in X.".format(distinct, K), ConvergenceWarning, stacklevel=2)
    return st.labels.to(torch.int64), st.out_centers, float(s[_lib.NNK_KM_INERTIA]), i + 1


class GaussianMixture(_SkGaussianMixture):
    """``sklearn.mixture.GaussianMixture`` whose EM runs on the GPU (csrc/nnk_gmm_em.cu).

    Same constructor, same fitted attributes (float64 NumPy arrays: ``weights_``, ``means_``,
    ``covariances_``, ``precisions_cholesky_``, ``precisions_``, ``converged_``, ``n_iter_``,
    ``lower_bound_``, ``lower_bounds_``), so scikit-learn's own ``predict``, ``predict_proba``, ``score``,
    ``sample``, ``bic``, pickling and this module's ``MLPG`` / ``MLPGBase`` work on the result.

    ``fit`` / ``fit_predict`` follow scikit-learn 1.9's ``BaseMixture.fit_predict`` step for step
    (``n_init``, ``warm_start``, ``max_iter=0``, the ``tol`` stop, ``ConvergenceWarning``, the final E-step
    whose arg-max gives the labels).  The initial responsibilities (``init_params`` in {"kmeans",
    "k-means++", "random", "random_from_data"}) come from scikit-learn on the host with the same
    ``random_state`` consumption, so the same seed gives the same start; the initial parameters are then
    computed from them on the device.  Only ``covariance_type="full"`` is supported, with at most 128
    features and 128 components.

    ``init_device`` (additive, default False): with ``init_params`` "kmeans" or "k-means++" the k-means
    initialisation runs on the GPU as well (csrc/nnk_kmeans.cu): scikit-learn's ``KMeans(n_init=1)`` /
    ``kmeans_plusplus`` restated step for step, consuming ``random_state`` the same way, in float64 on the
    frames widened to float64.  Only its labels (or seeds) cross into EM, so on the same labels the fit is
    bit-identical to ``init_device=False``.  "random" and "random_from_data" ignore it.

    ``X`` may be a NumPy array or a torch CUDA tensor, float32 or float64; a CUDA tensor is copied to
    the host only when a host initialiser ("kmeans", "k-means++" with ``init_device=False``) needs it, and
    ``fit_predict`` then returns the labels as a CUDA tensor.  The arithmetic is always float64.  Note that scikit-learn 1.9
    itself fits float32 data in float32, so on float32 input the two differ; this class matches
    scikit-learn run on the same data widened to float64 (to about 1e-10 relative: the summation order
    of the reductions differs in the last bits).
    """

    _parameter_constraints = {**_SkGaussianMixture._parameter_constraints, "init_device": ["boolean"]}

    def __init__(self, n_components=1, *, covariance_type="full", tol=1e-3, reg_covar=1e-6, max_iter=100, n_init=1,
                 init_params="kmeans", weights_init=None, means_init=None, precisions_init=None, random_state=None,
                 warm_start=False, verbose=0, verbose_interval=10, init_device=False):
        super().__init__(n_components=n_components, covariance_type=covariance_type, tol=tol, reg_covar=reg_covar,
                         max_iter=max_iter, n_init=n_init, init_params=init_params, weights_init=weights_init,
                         means_init=means_init, precisions_init=precisions_init, random_state=random_state,
                         warm_start=warm_start, verbose=verbose, verbose_interval=verbose_interval)
        self.init_device = init_device

    def _check_sizes(self, D):
        if self.covariance_type != "full":
            raise NotImplementedError("nnmnkwii_b200 GaussianMixture fits covariance_type='full' only (got %r)"
                                      % (self.covariance_type,))
        if D > _EM_MAX_FEATURES:
            raise ValueError("GaussianMixture on the GPU supports at most %d features (got %d)" % (_EM_MAX_FEATURES, D))
        if self.n_components > _EM_MAX_COMPONENTS:
            raise ValueError("GaussianMixture on the GPU supports at most %d components (got %d)"
                             % (_EM_MAX_COMPONENTS, self.n_components))

    def _initial_resp(self, n_samples, host_X, random_state):
        """The responsibilities scikit-learn's ``_initialize_parameters`` derives, computed the same way
        (same RandomState calls), in float64."""
        from sklearn import cluster
        from sklearn.cluster import kmeans_plusplus
        K = self.n_components
        resp = np.zeros((n_samples, K), dtype=np.float64)
        if self.init_params == "kmeans":
            label = cluster.KMeans(n_clusters=K, n_init=1, random_state=random_state).fit(host_X()).labels_
            resp[np.arange(n_samples), label] = 1
        elif self.init_params == "random":
            resp = np.asarray(random_state.uniform(size=(n_samples, K)), dtype=np.float64)
            resp /= np.sum(resp, axis=1)[:, np.newaxis]
        elif self.init_params == "random_from_data":
            indices = random_state.choice(n_samples, size=K, replace=False)
            for col, index in enumerate(indices):
                resp[index, col] = 1
        elif self.init_params == "k-means++":
            _, indices = kmeans_plusplus(host_X(), K, random_state=random_state)
            resp[indices, np.arange(K)] = 1
        return resp

    def _device_initial_resp(self, st, random_state):
        """``_initial_resp`` for "kmeans" / "k-means++" with the k-means on the device: the one-hot
        responsibilities are scattered into ``st.resp`` without a host copy of the frames."""
        import torch
        K = self.n_components
        st.resp.zero_()
        if self.init_params == "kmeans":
            labels, _, _, _ = _device_kmeans(st.X, K, random_state=random_state)
            st.resp.scatter_(1, labels[:, None], 1.0)
        else:
            _, indices = _device_kmeans_plusplus(st.X, K, random_state)
            st.resp[indices, torch.arange(K, device=st.resp.device)] = 1.0

    def _device_initialize(self, st, n_samples, host_X, random_state):
        """sklearn's ``GaussianMixture._initialize_parameters`` + ``_initialize``; returns whether the
        device covariances are valid (they are not when ``precisions_init`` is given)."""
        from sklearn.mixture._gaussian_mixture import _compute_precision_cholesky_from_precisions
        from sklearn.utils._array_api import get_namespace
        compute_resp = self.weights_init is None or self.means_init is None or self.precisions_init is None
        if compute_resp and self.init_device and self.init_params in ("kmeans", "k-means++"):
            self._device_initial_resp(st, random_state)
            st.mstep(0 if self.weights_init is None else 2)
        elif compute_resp:
            st.put("resp", self._initial_resp(n_samples, host_X, random_state))
            st.mstep(0 if self.weights_init is None else 2)
        if self.weights_init is not None:
            st.put("weights", self.weights_init)
        if self.means_init is not None:
            st.put("means", self.means_init)
        if self.precisions_init is None:
            st.factor(True)
            st.check_status()
            return True
        prec = np.asarray(self.precisions_init, dtype=np.float64)
        st.put("prec_chol", _compute_precision_cholesky_from_precisions(prec, self.covariance_type,
                                                                         xp=get_namespace(prec)[0]))
        st.factor(False)
        return False

    def fit_predict(self, X, y=None):
        """Estimate the model parameters with EM on the GPU and return the labels of ``X``.

        Mirrors ``sklearn.mixture.GaussianMixture.fit_predict`` (see the class docstring)."""
        import warnings

        import torch
        from sklearn.exceptions import ConvergenceWarning
        from sklearn.utils import check_random_state
        from sklearn.utils._array_api import get_namespace

        self._validate_params()
        Xd, Xh = _as_frames(X)
        n_samples, D = Xd.shape
        self._check_sizes(D)
        if n_samples < self.n_components:
            raise ValueError("Expected n_samples >= n_components but got n_components = %d, n_samples = %d"
                             % (self.n_components, n_samples))
        self.n_features_in_ = D
        if hasattr(self, "feature_names_in_"):
            del self.feature_names_in_
        shape_only = np.empty((0, D))  # sklearn's _check_parameters reads X.shape only
        self._check_parameters(shape_only, xp=get_namespace(shape_only)[0])

        cache = {}

        def host_X():
            if "X" not in cache:
                cache["X"] = np.asarray(Xh, dtype=np.float64) if Xh is not None else _host_f64(Xd)
            return cache["X"]

        st = _EmState(Xd, self.n_components, self.reg_covar)
        do_init = not (self.warm_start and hasattr(self, "converged_"))
        n_init = self.n_init if do_init else 1
        max_lower_bound = -np.inf
        best_lower_bounds = []
        best = None
        self.converged_ = False
        random_state = check_random_state(self.random_state)
        cov_valid = False
        if not do_init:  # warm start: continue from the fitted attributes
            st.put("weights", self.weights_)
            st.put("means", self.means_)
            st.put("prec_chol", self.precisions_cholesky_)
            if getattr(self, "covariances_", None) is not None:
                st.put("covariances", self.covariances_)
                cov_valid = True
            st.factor(False)

        def snapshot():
            return (st.weights.clone(), st.means.clone(), st.covariances.clone() if cov_valid else None,
                    st.prec_chol.clone())

        for init in range(n_init):
            self._print_verbose_msg_init_beg(init)
            if do_init:
                cov_valid = self._device_initialize(st, n_samples, host_X, random_state)
            lower_bound = -np.inf if do_init else self.lower_bound_
            current_lower_bounds = []
            if self.max_iter == 0:
                best = snapshot()
                best_n_iter = 0
            else:
                converged = False
                for n_iter in range(1, self.max_iter + 1):
                    prev_lower_bound = lower_bound
                    st.estep()
                    st.mstep(1)
                    st.factor(True)
                    cov_valid = True
                    st.check_status()
                    lower_bound = float(st.lower_bound.item())
                    current_lower_bounds.append(lower_bound)
                    change = lower_bound - prev_lower_bound
                    self._print_verbose_msg_iter_end(n_iter, change)
                    if abs(change) < self.tol:
                        converged = True
                        break
                self._print_verbose_msg_init_end(lower_bound, converged)
                if lower_bound > max_lower_bound or max_lower_bound == -np.inf:
                    max_lower_bound = lower_bound
                    best = snapshot()
                    best_n_iter = n_iter
                    best_lower_bounds = current_lower_bounds
                    self.converged_ = converged

        if not self.converged_ and self.max_iter > 0:
            warnings.warn("Best performing initialization did not converge. Try different init parameters, or "
                          "increase max_iter, tol, or check for degenerate data.", ConvergenceWarning)

        w, m, c, pc = best
        # like sklearn's _get_parameters: without a covariance estimate (precisions_init, max_iter=0) the
        # attribute keeps whatever it was, and is missing on a fresh estimator
        cov_host = _host_f64(c) if c is not None else self.covariances_
        self._set_parameters((_host_f64(w), _host_f64(m), cov_host, _host_f64(pc)))
        self.n_iter_ = best_n_iter
        self.lower_bound_ = max_lower_bound
        self.lower_bounds_ = best_lower_bounds

        # final E-step with the kept parameters: labels consistent with fit(X).predict(X)
        st.weights.copy_(w)
        st.means.copy_(m)
        st.prec_chol.copy_(pc)
        st.factor(False)
        st.estep()
        labels = torch.argmax(st.resp, dim=1)
        if Xh is None:
            return labels
        return labels.cpu().numpy()


__all__ = ["MLPGBase", "MLPG", "GaussianMixture"]
