"""Without a GPU: the catalogue of tests/test_buffers_and_streams_gpu.py names every public entry point of the
kernel-launching modules (or says why one needs no case), and sorts every C-ABI symbol."""
import importlib

import stream_catalogue as C


def _public(modname):
    mod = importlib.import_module("nnmnkwii_b200." + modname)
    names = getattr(mod, "__all__", None)
    if names is None:
        names = [n for n, v in vars(mod).items()
                 if not n.startswith("_") and callable(v) and getattr(v, "__module__", "") == mod.__name__]
    return {(modname, n) for n in names if callable(getattr(mod, n))}


def test_every_public_entry_point_is_catalogued_or_host_only():
    public = set()
    for m in C.MODULES:
        public |= _public(m)
    missing = sorted(public - C.COVERED - set(C.HOST_ONLY))
    assert not missing, "public entry points with neither a case nor a host-only reason: %s" % missing
    assert not (C.COVERED & set(C.HOST_ONLY)), sorted(C.COVERED & set(C.HOST_ONLY))
    stale = sorted((C.COVERED | set(C.HOST_ONLY)) - public)
    assert not stale, "catalogued names that are not public: %s" % stale
    assert all(r.strip() for r in C.HOST_ONLY.values())


def test_every_export_is_sorted():
    from nnmnkwii_b200 import _lib
    exports = set(_lib.EXPORTS)
    assert set(C.EXPORTS_NOT_LAUNCHING) <= exports and C.EXPORTS_SHARDING <= exports
    assert not (set(C.EXPORTS_NOT_LAUNCHING) & C.EXPORTS_SHARDING)
    launching = C.launching_exports(exports)
    # the symbols the kernel families launch through, by header name
    for name in ("nnk_mlpg_fwd", "nnk_mlpg_grad", "nnk_mlpg_solve", "nnk_mlpg_gv", "nnk_dtw_align",
                 "nnk_postfilter_apply", "nnk_gmm_em_estep", "nnk_kmeans_seed", "nnk_mlpg_host", "nnk_modspec",
                 "nnk_gmm_traj_em", "nnk_mlpg_ms", "nnk_mlpg_ms_segment", "nnk_ms_segment", "nnk_mix_gen",
                 "nnk_mlpg_traj_ll", "nnk_mlpg_traj_sample", "nnk_mlpg_vjp"):
        assert name in launching, name
    assert not any(n.endswith("_workspace_bytes") for n in launching)


def test_every_launching_export_takes_the_stream_last():
    """The GPU module reads a launching call's stream from its last argument; the exceptions run their own."""
    import ctypes

    from test_abi import prototypes

    from nnmnkwii_b200 import _lib
    launching = C.launching_exports(_lib.EXPORTS)
    assert C.EXPORTS_OWN_STREAMS <= set(launching)
    params = {name: p for _, name, p in prototypes()}
    for name in launching:
        if name not in C.EXPORTS_OWN_STREAMS:
            assert _lib.SIGNATURES[name][1][-1] is ctypes.c_void_p, name
            assert params[name][-1] == "void* stream", name
