"""Host side of UnitVarianceMLPG: reduce the dense MLPG matrix R to its numerical band (once per R,
cached) and enqueue the stencil sweeps of csrc/nnk_uvmlpg.cu.  No arithmetic on the host."""
import ctypes
import weakref

import torch

from . import _device as dev
from . import _lib
from ._lib import lib

# relative magnitude (w.r.t. max |R|) below which off-band entries of R are dropped.  A float32 R has
# resolution 6e-8 (2^-24): everything dropped sums to well below that.  A float64 R is only cut where
# its entries are below ITS resolution.  K = T - 1 reproduces R exactly (an arbitrary dense R simply
# gets K = T - 1 and the per-row table kernels: nothing is ever silently banded).
BAND_REL_TOL = {"float32": 2.0 ** -32, "float64": 2.0 ** -60}

_band_cache = {}


# rows whose band differs from the middle row by less than this (relative to max |R|) share its filter.
# R's own float32 rounding makes two copies of the same filter differ by up to 2^-24 max|R| per entry, so
# 2^-23 is the tightest test that still recognises the shift-invariant rows; per output the substitution
# error is then bounded by (2K+1) nw 2^-23 max|R| max|x| (5e-5 at K = 23) and is ~ sqrt of that count in
# practice, the level of the float32 rounding of R itself.  float32 R only.
TOEPLITZ_REL_TOL = 2.0 ** -23
TOEPLITZ_MIN_ROWS = 64
# h_w = h_0 * c_w fit (factored sweep): accepted when the residual is below the same resolution
FACTOR_REL_TOL = 2.0 ** -23


class Band(object):
    __slots__ = ("Rb", "RbT", "K", "T", "nw", "dtype", "toep", "toepT", "fact", "factT")


def _toeplitz_interval(table, peak):
    """(t_lo, t_hi, taps) of the maximal run of rows around T//2 equal to the middle row (host side,
    once per R): table is the (T, nw, 2K+1) band table."""
    import numpy as np
    tab = table.cpu().numpy()
    T = tab.shape[0]
    mid = T // 2
    ok = np.abs(tab - tab[mid]).reshape(T, -1).max(axis=1) <= peak * TOEPLITZ_REL_TOL
    lo = mid
    while lo > 0 and ok[lo - 1]:
        lo -= 1
    hi = mid + 1
    while hi < T and ok[hi]:
        hi += 1
    return lo, hi, np.ascontiguousarray(tab[mid], dtype=np.float32)


def _factor_taps(taps, K, peak):
    """Short stencils c_w (nw, 2*KC+1) with  taps[w] = taps[0] * c_w  (h_w[j] = sum_k c_w[k] h_0[j - k + KC]),
    KC in (1, 2), by least squares on the band row; None if the residual exceeds FACTOR_REL_TOL * peak
    (e.g. an R that is not an MLPG matrix).  Host side, once per R."""
    import numpy as np
    h = np.asarray(taps, dtype=np.float64)
    nw, W = h.shape
    if nw < 2 or nw > 3 or K > 32:
        return None
    for KC in (1, 2):
        A = np.zeros((W, 2 * KC + 1))
        for k in range(2 * KC + 1):
            for j in range(W):
                i = j - k + KC
                if 0 <= i < W:
                    A[j, k] = h[0, i]
        c = np.zeros((nw, 2 * KC + 1))
        good = True
        for w in range(nw):
            sol = np.linalg.lstsq(A, h[w], rcond=None)[0]
            if np.abs(A @ sol - h[w]).max() > peak * FACTOR_REL_TOL:
                good = False
                break
            c[w] = sol
        if good:
            return KC, np.ascontiguousarray(h[0], dtype=np.float32), np.ascontiguousarray(c, dtype=np.float32)
    return None


def band_of(R, device):
    """Band tables of R (cached on (data_ptr, version, shape, device)).  The caller reads them on the
    current stream of ``device``; an eviction never recycles their blocks before those reads have run."""
    assert R.dim() == 2 and R.shape[1] % R.shape[0] == 0
    key = (R.data_ptr(), R._version, tuple(R.shape), R.dtype, str(R.device), str(device))
    hit = _band_cache.get(key)
    if hit is not None and hit[0]() is R:
        dev.keep_for_current_stream(hit[1].Rb, device)
        dev.keep_for_current_stream(hit[1].RbT, device)
        return hit[1]
    Rd = R.detach().to(device)
    if Rd.dtype not in (torch.float32, torch.float64):
        Rd = Rd.to(torch.float32)
    Rd = Rd.contiguous()
    T = Rd.shape[0]
    nw = Rd.shape[1] // T
    code = dev.torch_dtype_code(Rd.dtype)
    stream = dev.current_stream_ptr(device)
    profile = torch.empty(T, dtype=torch.float32, device=device)
    _lib.check(lib.nnk_uv_band_profile(Rd.data_ptr(), code, T, nw, profile.data_ptr(), stream), "nnk_uv_band_profile")
    prof = profile.cpu()
    peak = float(prof.max())
    above = torch.nonzero(prof > peak * BAND_REL_TOL["float64" if Rd.dtype == torch.float64 else "float32"])
    K = int(above.max()) if above.numel() else 0
    b = Band()
    b.K, b.T, b.nw, b.dtype = K, T, nw, Rd.dtype
    b.Rb = torch.empty((T, nw, 2 * K + 1), dtype=Rd.dtype, device=device)
    b.RbT = torch.empty((T, nw, 2 * K + 1), dtype=Rd.dtype, device=device)
    _lib.check(lib.nnk_uv_band_extract(Rd.data_ptr(), code, T, nw, K, b.Rb.data_ptr(), b.RbT.data_ptr(), stream),
               "nnk_uv_band_extract")
    b.toep = b.toepT = b.fact = b.factT = None
    if Rd.dtype == torch.float32 and nw <= 3 and K <= 64 and T >= TOEPLITZ_MIN_ROWS:
        lo, hi, taps = _toeplitz_interval(b.Rb, peak)
        if hi - lo >= TOEPLITZ_MIN_ROWS:
            b.toep = (lo, hi, taps)
            b.fact = _factor_taps(taps, K, peak)
        lo, hi, taps = _toeplitz_interval(b.RbT, peak)
        if hi - lo >= TOEPLITZ_MIN_ROWS:
            b.toepT = (lo, hi, taps)
            b.factT = _factor_taps(taps, K, peak)
    if len(_band_cache) > 16:
        _band_cache.clear()
    try:
        _band_cache[key] = (weakref.ref(R), b)
    except TypeError:
        pass
    return b


def apply_forward(band, means3, reshaped):
    """means3: (B, T, nw*sd) [reshaped=False] or (B, nw*T, sd) [reshaped=True] -> (B, T, sd)."""
    B = means3.shape[0]
    T, nw = band.T, band.nw
    if reshaped:
        assert means3.shape[1] == nw * T
        sd = means3.shape[2]
    else:
        assert means3.shape[1] == T
        sd = means3.shape[2] // nw
        if means3.shape[2] != nw * sd:
            means3 = means3[..., : nw * sd]
    x = means3.to(band.dtype).contiguous()
    y = torch.empty((B, T, sd), dtype=band.dtype, device=x.device)
    if band.toep is not None and band.fact is not None:
        lo, hi, _ = band.toep
        kc, h0, c = band.fact
        _lib.check(lib.nnk_uv_apply_factored(band.Rb.data_ptr(), h0.ctypes.data, c.ctypes.data, x.data_ptr(), y.data_ptr(),
                                             B, T, sd, nw, band.K, kc, lo, hi, 0, int(reshaped),
                                             dev.current_stream_ptr(x.device)), "nnk_uv_apply_factored")
    elif band.toep is not None:
        lo, hi, taps = band.toep
        _lib.check(lib.nnk_uv_apply_toeplitz(band.Rb.data_ptr(), taps.ctypes.data, x.data_ptr(), y.data_ptr(), B, T, sd, nw,
                                             band.K, lo, hi, 0, int(reshaped), dev.current_stream_ptr(x.device)),
                   "nnk_uv_apply_toeplitz")
    else:
        _lib.check(lib.nnk_uv_apply(band.Rb.data_ptr(), x.data_ptr(), y.data_ptr(), dev.torch_dtype_code(band.dtype),
                                    B, T, sd, nw, band.K, 0, int(reshaped), dev.current_stream_ptr(x.device)), "nnk_uv_apply")
    return y.to(means3.dtype) if y.dtype != means3.dtype else y


def apply_backward(band, grad_output3, reshaped, D):
    """grad_output3: (B, T, sd) -> gradient w.r.t. means: (B, nw*T, sd) or (B, T, D)."""
    B, T, sd = grad_output3.shape
    nw = band.nw
    assert T == band.T
    g = grad_output3.to(band.dtype).contiguous()
    if reshaped:
        gx = torch.empty((B, nw * T, sd), dtype=band.dtype, device=g.device)
    else:
        gx = torch.empty((B, T, nw * sd), dtype=band.dtype, device=g.device)
    if band.toepT is not None and band.factT is not None:
        lo, hi, _ = band.toepT
        kc, h0, c = band.factT
        _lib.check(lib.nnk_uv_apply_factored(band.RbT.data_ptr(), h0.ctypes.data, c.ctypes.data, g.data_ptr(), gx.data_ptr(),
                                             B, T, sd, nw, band.K, kc, lo, hi, 1, int(reshaped),
                                             dev.current_stream_ptr(g.device)), "nnk_uv_apply_factored")
    elif band.toepT is not None:
        lo, hi, taps = band.toepT
        _lib.check(lib.nnk_uv_apply_toeplitz(band.RbT.data_ptr(), taps.ctypes.data, g.data_ptr(), gx.data_ptr(), B, T, sd, nw,
                                             band.K, lo, hi, 1, int(reshaped), dev.current_stream_ptr(g.device)),
                   "nnk_uv_apply_toeplitz")
    else:
        _lib.check(lib.nnk_uv_apply(band.RbT.data_ptr(), g.data_ptr(), gx.data_ptr(), dev.torch_dtype_code(band.dtype),
                                    B, T, sd, nw, band.K, 1, int(reshaped), dev.current_stream_ptr(g.device)), "nnk_uv_apply")
    if not reshaped and nw * sd != D:  # trailing columns the forward ignored get zero gradient
        full = torch.zeros((B, T, D), dtype=band.dtype, device=g.device)
        full[..., : nw * sd] = gx
        gx = full
    return gx.to(grad_output3.dtype) if gx.dtype != grad_output3.dtype else gx


_ = ctypes
