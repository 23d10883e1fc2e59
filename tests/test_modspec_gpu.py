"""Modulation spectrum on the GPU: preprocessing.modspec / modphase / inv_modspec / modspec_smoothing and
autograd.ModSpec / ModSpecBatch.

* the reference's outputs (tests/golden/modspec_reference_golden.npz, written by make_modspec_golden.py) at every
  DFT length, T = 1, odd, n - 1 and n, norm None and "ortho": float64 within 1e-10, float32 within 1e-4;
* torch.fft as a second oracle on whole outputs, D = 1 and 37, every norm;
* the round trip, smoothing above the Nyquist frequency (the identity) and smoothing twice (idempotent);
* a padded batch with NaN in its padding equals per-utterance calls bit for bit;
* gradcheck of the float64 gradient, and the float32 gradient against it.

Dirty allocations, workspace reuse and a delayed side stream are checked for these entry points by the
buffers-and-streams catalogue (tests/test_buffers_and_streams_gpu.py), as for every other one."""
import importlib.util
import os

import numpy as np
import pytest

from conftest import ROOT, rel_err

pytestmark = pytest.mark.gpu

_spec = importlib.util.spec_from_file_location("make_modspec_golden",
                                               os.path.join(ROOT, "tests", "golden", "make_modspec_golden.py"))
MG = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(MG)
TOL = {np.float64: 1e-10, np.float32: 1e-4}


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "modspec_reference_golden.npz"))


def _np(t):
    return t.detach().cpu().numpy()


def _crel(a, b):
    """max |a - b| / max |b| of complex arrays."""
    a, b = np.asarray(a, np.complex128), np.asarray(b, np.complex128)
    return float(np.abs(a - b).max() / max(1e-300, np.abs(b).max()))


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("n", MG.NS)
def test_reference_parity(golden, n, dtype):
    import torch

    from nnmnkwii_b200 import preprocessing as P
    tol = TOL[dtype]
    for nn, T, D, seed in MG.cases():
        if nn != n:
            continue
        x = torch.from_numpy(MG.trajectory(T, D, seed).astype(dtype)).cuda()
        kb, kt, kn = MG.pick(n // 2 + 1), MG.pick(T), MG.pick(n)
        for norm in MG.NORMS:
            tag = (n, T, norm)
            ms, ph = P.modspec(x, n=n, norm=norm, return_phase=True)
            assert ms.dtype == x.dtype and ph.dtype == (torch.complex128 if dtype == np.float64 else torch.complex64)
            r_ms, r_ph = golden[MG.key("ms", *tag)], golden[MG.key("phase", *tag)]
            assert rel_err(_np(ms)[kb], r_ms) <= tol, tag
            if dtype == np.float64:
                assert _crel(_np(ph)[kb], r_ph) <= tol, tag
            else:  # float32 phase is judged where it matters, weighted by the amplitude
                assert _crel(np.sqrt(_np(ms)[kb]) * _np(ph)[kb], np.sqrt(r_ms) * r_ph) <= tol, tag
            assert torch.equal(P.modphase(x, n=n, norm=norm), ph)
            assert rel_err(_np(P.inv_modspec(ms, ph, norm=norm))[kn], golden[MG.key("inv", *tag)]) <= tol, tag
            sm = P.modspec_smoothing(x, MG.MODFS, n=n, norm=norm, cutoff=MG.CUTOFF)
            assert sm.shape == x.shape and rel_err(_np(sm)[kt], golden[MG.key("smooth", *tag)]) <= tol, tag
            if norm is None:
                sl = P.modspec_smoothing(x, MG.MODFS, n=n, norm=norm, cutoff=MG.CUTOFF, log_domain=False)
                assert rel_err(_np(sl)[kt], golden[MG.key("smoothlin", *tag)]) <= tol, tag
    # NumPy in, NumPy out
    x = MG.trajectory(n // 4 + 1, 3, 1).astype(dtype)
    ms = P.modspec(x, n=n)
    assert isinstance(ms, np.ndarray) and ms.dtype == dtype and ms.shape == (n // 2 + 1, 3)


def _torch_oracle(x64, n, norm, modfs, cutoff, log_domain):
    """(power, phase, smoothed) of a float64 (T, D) CUDA tensor by torch.fft."""
    import torch
    X = torch.fft.rfft(x64, n=n, dim=0, norm=norm)
    pw = X.real ** 2 + X.imag ** 2
    ph = torch.exp(1j * torch.angle(X))
    ms = torch.log(pw) if log_domain else pw.clone()
    ms[int(n * cutoff / modfs) + 1:] = 0
    if log_domain:
        ms = torch.exp(ms)
    return pw, ph, torch.fft.irfft(torch.sqrt(ms) * ph, n=n, dim=0, norm=norm)[:x64.shape[0]]


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("n", MG.NS)
def test_against_torch_fft(n, dtype):
    import torch

    from nnmnkwii_b200 import preprocessing as P
    tol = TOL[dtype]
    g = torch.Generator(device="cuda").manual_seed(n)
    for T in (1, 7, n - 1, n):
        for D in (1, 37):
            x64 = torch.randn((T, D), dtype=torch.float64, device="cuda", generator=g).cumsum(0) * 0.1
            x = x64.to(getattr(torch, np.dtype(dtype).name))
            for norm in (None, "ortho", "forward"):
                for log_domain in (True, False):
                    pw, ph, sm = _torch_oracle(x.double(), n, norm, 200, 30, log_domain)
                    ms, mph = P.modspec(x, n=n, norm=norm, return_phase=True)
                    tag = (T, D, norm, log_domain)
                    assert rel_err(_np(ms), _np(pw)) <= tol, tag
                    assert _crel(_np(ms.sqrt() * mph), _np(pw.sqrt() * ph)) <= tol, tag
                    out = P.modspec_smoothing(x, 200, n=n, norm=norm, cutoff=30, log_domain=log_domain)
                    assert rel_err(_np(out), _np(sm)) <= tol, tag
                    inv = P.inv_modspec(ms, mph, norm=norm)
                    assert inv.shape == (n, D)
                    assert rel_err(_np(inv), _np(torch.fft.irfft(pw.sqrt() * ph, n=n, dim=0, norm=norm))) <= tol, tag


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("norm", [None, "ortho"])
def test_round_trip(norm, dtype):
    import torch

    from nnmnkwii_b200 import preprocessing as P
    rng = np.random.default_rng(3)
    for n in MG.NS:
        for T in (1, 100, n):
            x = torch.from_numpy(rng.standard_normal((T, 5)).astype(dtype)).cuda()
            back = P.inv_modspec(*P.modspec(x, n=n, norm=norm, return_phase=True), norm=norm)[:T]
            assert rel_err(_np(back), _np(x)) <= TOL[dtype], (n, T)
    lens = [300, 1, 512, 77]
    xb = torch.from_numpy(rng.standard_normal((4, 512, 3)).astype(dtype)).cuda()
    ms, ph = P.modspec(xb, n=1024, norm=norm, return_phase=True, lengths=lens)
    back = P.inv_modspec(ms, ph, norm=norm, lengths=lens)
    assert back.shape == xb.shape
    for b, L in enumerate(lens):
        assert rel_err(_np(back[b, :L]), _np(xb[b, :L])) <= TOL[dtype] and not back[b, L:].any()


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_smoothing_invariants(dtype):
    """Smoothing with the cut-off at the Nyquist frequency (or none) keeps every band: the identity on the T
    frames.  Smoothing twice equals smoothing once when T = n; for T < n the output is cut to T frames and
    zero-padded again before the second pass, which is a different trajectory."""
    import torch

    from nnmnkwii_b200 import preprocessing as P
    rng = np.random.default_rng(4)
    for n in MG.NS:
        for T in (1, 123, n):
            x = torch.from_numpy(rng.standard_normal((T, 4)).astype(dtype)).cuda()
            for log_domain in (True, False):
                for cutoff in (100, None):
                    y = P.modspec_smoothing(x, 200, n=n, cutoff=cutoff, log_domain=log_domain)
                    assert rel_err(_np(y), _np(x)) <= TOL[dtype], (n, T, log_domain, cutoff)
        x = torch.from_numpy(rng.standard_normal((n, 4)).astype(dtype)).cuda()
        for log_domain in (True, False):
            for norm in (None, "ortho"):
                once = P.modspec_smoothing(x, 200, n=n, norm=norm, cutoff=20, log_domain=log_domain)
                twice = P.modspec_smoothing(once, 200, n=n, norm=norm, cutoff=20, log_domain=log_domain)
                assert rel_err(_np(twice), _np(once)) <= TOL[dtype], (n, log_domain, norm)
                assert rel_err(_np(once), _np(x)) > 1e-2  # the smoothing did remove something


# ---- batched == per utterance, whatever the padding ------------------------------------------------------------------
def _all_outputs(xb, lens, n, norm, grad_ms):
    """Every entry point on a padded batch: the list of its results."""
    from nnmnkwii_b200 import preprocessing as P
    from nnmnkwii_b200.preprocessing.modspec import _modspec_grad
    ms, ph = P.modspec(xb, n=n, norm=norm, return_phase=True, lengths=lens)
    return [ms, ph, P.modspec(xb, n=n, norm=norm, lengths=lens),
            P.modspec_smoothing(xb, 200, n=n, norm=norm, cutoff=40, lengths=lens),
            P.modspec_smoothing(xb, 200, n=n, norm=norm, cutoff=40, log_domain=False, lengths=lens),
            P.inv_modspec(ms, ph, norm=norm, lengths=lens), P.inv_modspec(ms, ph, norm=norm),
            _modspec_grad(xb, grad_ms, n, norm, lens)]


def _same(a, b):
    import torch
    return a.shape == b.shape and torch.equal(torch.view_as_real(a) if a.is_complex() else a,
                                              torch.view_as_real(b) if b.is_complex() else b)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("n", [256, 4096])
def test_batched_equals_per_utterance(n, dtype):
    import torch

    from nnmnkwii_b200 import preprocessing as P
    from nnmnkwii_b200.preprocessing.modspec import _modspec_grad
    rng = np.random.default_rng(n)
    T, D, norm = min(n, 300), 7, "ortho"
    lens = np.array([T, 1, 0, T // 2 + 1, 17])
    tdt = getattr(torch, np.dtype(dtype).name)
    utts = [torch.from_numpy(rng.standard_normal((L, D)).astype(dtype)).cuda() for L in lens]
    G = torch.from_numpy(rng.standard_normal((len(lens), n // 2 + 1, D)).astype(dtype)).cuda()
    # per utterance, plain
    want = []
    for b, u in enumerate(utts):
        ms, ph = P.modspec(u, n=n, norm=norm, return_phase=True)
        want.append([ms, ph, P.modspec(u, n=n, norm=norm),
                     P.modspec_smoothing(u, 200, n=n, norm=norm, cutoff=40),
                     P.modspec_smoothing(u, 200, n=n, norm=norm, cutoff=40, log_domain=False),
                     P.inv_modspec(ms, ph, norm=norm)[:len(u)], P.inv_modspec(ms, ph, norm=norm),
                     _modspec_grad(u, G[b], n, norm)])
    padded = torch.full((len(lens), T, D), float("nan"), dtype=tdt, device="cuda")
    for b, u in enumerate(utts):
        padded[b, :len(u)] = u

    def check(got):
        for b, L in enumerate(lens):
            for i, (g, w) in enumerate(zip(got, want[b])):
                if i in (3, 4, 5, 7):  # frame outputs: the utterance's frames, then zeros
                    assert _same(g[b, :L], w[:L]) and not g[b, L:].any(), (b, i)
                else:
                    assert _same(g[b], w), (b, i)

    check(_all_outputs(padded, lens, n, norm, G))


# ---- gradients ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("norm", [None, "ortho", "forward"])
def test_gradcheck(norm):
    import torch

    from nnmnkwii_b200 import autograd as A
    torch.manual_seed(0)
    y = torch.randn(9, 2, dtype=torch.float64, device="cuda", requires_grad=True)
    assert torch.autograd.gradcheck(lambda v: A.modspec(v, 256, norm), (y,), eps=1e-6, atol=1e-7, rtol=1e-6)
    yb = torch.randn(3, 9, 2, dtype=torch.float64, device="cuda", requires_grad=True)
    lens = [9, 4, 1]
    assert torch.autograd.gradcheck(lambda v: A.modspec_batch(v, lens, 256, norm), (yb,), eps=1e-6, atol=1e-7,
                                    rtol=1e-6)
    yb.grad = None
    A.modspec_batch(yb, lens, 256, norm).sum().backward()
    for b, L in enumerate(lens):
        assert not yb.grad[b, L:].any()


@pytest.mark.parametrize("n", [512, 4096])
def test_float32_gradient_matches_float64(n):
    import torch

    from nnmnkwii_b200 import autograd as A
    rng = np.random.default_rng(5)
    x = rng.standard_normal((200, 6)).cumsum(0) * 0.1
    target = rng.standard_normal((n // 2 + 1, 6)) ** 2
    grads = {}
    for dt in (torch.float64, torch.float32):
        y = torch.tensor(x, dtype=dt, device="cuda", requires_grad=True)
        ms = A.modspec(y, n, "ortho")
        assert ms.dtype == dt
        ((ms.log1p() - torch.tensor(target, dtype=dt, device="cuda").log1p()) ** 2).sum().backward()
        grads[dt] = _np(y.grad).astype(np.float64)
    assert rel_err(grads[torch.float32], grads[torch.float64]) <= 1e-4
    # the reference's dense formula, float64: 2 C (R cos + I sin) with kt = -2 pi k t / n
    y = torch.tensor(x, device="cuda", requires_grad=True)
    G = torch.from_numpy(rng.standard_normal((n // 2 + 1, 6))).cuda()
    (A.modspec(y, n, None) * G).sum().backward()
    X = np.fft.rfft(x, n=n, axis=0)
    kt = -2 * np.pi / n * np.arange(n // 2 + 1)[:, None] * np.arange(200)
    dense = np.stack([_np(G)[:, d] @ (2 * (X.real[:, d, None] * np.cos(kt) + X.imag[:, d, None] * np.sin(kt)))
                      for d in range(6)], axis=1)
    assert rel_err(_np(y.grad), dense) <= 1e-10
