"""CPU: the C-ABI library builds, loads and exports every symbol include/nnk_b200.h declares; the binding
(nnmnkwii_b200/_lib.py) matches every prototype, struct and integer constant of that header; and the product
never routes through the oracle or any CPU fallback.  No compute calls (no GPU here)."""
import ctypes
import os
import re

import pytest

from conftest import ROOT


def _header():
    return open(os.path.join(ROOT, "include", "nnk_b200.h")).read()


def test_library_exports_every_declared_symbol():
    from nnmnkwii_b200 import _lib
    declared = sorted(set(re.findall(r"\b(nnk_[a-z0-9_]+)\s*\(", _header())))
    assert len(declared) >= 10
    L = ctypes.CDLL(_lib.LIB_PATH)
    for name in declared:
        assert hasattr(L, name), "libnnk_b200.so does not export %s" % name
    assert sorted(_lib.EXPORTS) == declared
    assert _lib.lib.nnk_abi_version() == int(re.search(r"#define NNK_ABI_VERSION (\d+)", _header()).group(1))


def _code():
    """The header without its comments."""
    return re.sub(r"/\*.*?\*/|//[^\n]*", "", _header(), flags=re.S)


def prototypes():
    """(return type, name, [parameter declarations]) of every function the header declares."""
    protos = re.findall(r"([A-Za-z_][\w ]*\**)\s*\b(nnk_[a-z0-9_]+)\s*\(([^()]*)\)\s*;", _code())
    return [(ret, name, [] if params.strip() in ("", "void") else [p.strip() for p in params.split(",")])
            for ret, name, params in protos]


def _c_kind(c_type):
    """'ptr', 'i4', 'i8', 'f8', 'struct nnk_<x>' or None (void) of a C type."""
    if "*" in c_type:
        return "ptr"
    c_type = c_type.replace("const", "").strip()
    if re.fullmatch(r"nnk_\w+_t", c_type):
        return "struct " + c_type[:-2]
    return {"void": None, "int": "i4", "int32_t": "i4", "int64_t": "i8", "uint64_t": "i8", "size_t": "i8",
            "double": "f8"}[c_type]


def _ctypes_kind(t):
    if t is None:
        return None
    if issubclass(t, (ctypes._Pointer, ctypes.c_void_p, ctypes.c_char_p)):
        return "ptr"
    if issubclass(t, ctypes.Array):
        return ("array", t._length_, _ctypes_kind(t._type_))
    if issubclass(t, ctypes.Structure):
        return "struct " + re.sub(r"(?<!^)([A-Z])", r"_\1", t.__name__).lower()
    if t is ctypes.c_double:
        return "f8"
    return "i%d" % ctypes.sizeof(t)


def test_signature_table_matches_header_prototypes():
    """Every binding has the header's arity and, per argument and result, the same kind: an int32_t bound
    as an int64_t (or back) would silently truncate or misread the argument."""
    from nnmnkwii_b200 import _lib
    protos = prototypes()
    assert sorted(name for _, name, _ in protos) == sorted(_lib.SIGNATURES)
    for ret, name, params in protos:
        restype, argtypes = _lib.SIGNATURES[name]
        assert _ctypes_kind(restype) == _c_kind(ret), name
        assert [_ctypes_kind(t) for t in argtypes] == [_c_kind(p.rsplit(None, 1)[0]) for p in params], name


def _struct_fields(body, _lib):
    """[(name, kind)] of the fields of a C struct body; an array's kind is ('array', length, element kind)."""
    fields = []
    for decl in (d.strip() for d in body.split(";")):
        if not decl:
            continue
        c_type, declarators = re.match(r"((?:const\s+)?[A-Za-z_]\w*\s*\**)\s*(.*)", decl, re.S).groups()
        for d in declarators.split(","):
            name = re.match(r"\s*(\**)\s*([A-Za-z_]\w*)", d).group(2)
            kind = _c_kind(c_type + ("*" if d.strip().startswith("*") else ""))
            for dim in reversed(re.findall(r"\[\s*(\w+)\s*\]", d)):
                kind = ("array", int(dim) if dim.isdigit() else getattr(_lib, dim), kind)
            fields.append((name, kind))
    return fields


def test_every_struct_matches_its_binding():
    """Each ``typedef struct nnk_<x> { ... } nnk_<x>_t`` has the fields of its ctypes class ``_lib.Nnk<X>`` (of
    ``CHAIN_DTYPE`` for nnk_chain) in the same order and of the same kinds, so both sides lay it out alike; and
    every ctypes structure of the binding is one of them."""
    from nnmnkwii_b200 import _lib
    structs = re.findall(r"typedef struct (nnk_\w+) \{(.*?)\} (\w+);", _code(), re.S)
    assert len(structs) >= 10
    bound = set()
    for name, body, alias in structs:
        assert alias == name + "_t", alias
        want = _struct_fields(body, _lib)
        if name == "nnk_chain":
            dt = _lib.CHAIN_DTYPE
            got = [(f, "i%d" % dt.fields[f][0].itemsize) for f in dt.names if dt.fields[f][0].kind == "i"]
        else:
            cls = getattr(_lib, "".join(p.capitalize() for p in name.split("_")))
            bound.add(cls.__name__)
            got = [(f, _ctypes_kind(t)) for f, t in cls._fields_]
        assert got == want, (name, got, want)
    structures = {n for n, v in vars(_lib).items() if isinstance(v, type) and issubclass(v, ctypes.Structure)}
    assert structures == bound, sorted(structures ^ bound)


def test_every_integer_constant_matches_its_binding():
    from nnmnkwii_b200 import _lib
    defines = re.findall(r"^#define (NNK_[A-Z0-9_]+)\s+(-?\d+)\b", _code(), re.M)
    assert len(defines) >= 25
    for name, value in defines:
        assert getattr(_lib, "ABI_VERSION" if name == "NNK_ABI_VERSION" else name) == int(value), name


def test_struct_layouts_match_header():
    from nnmnkwii_b200 import _lib
    assert ctypes.sizeof(_lib.NnkWindows) == 4 + 4 * _lib.NNK_MAX_WIN * 2 + 4 + 8 * _lib.NNK_MAX_WIN * _lib.NNK_MAX_TAPS
    assert ctypes.sizeof(_lib.NnkStatus) == 16
    assert _lib.CHAIN_DTYPE.itemsize == 16


def test_status_decode_roundtrip():
    from nnmnkwii_b200 import _lib
    st = _lib.NnkStatus()
    _lib.lib.nnk_status_decode(ctypes.c_uint64(0), ctypes.byref(st))
    assert st.code == 0
    key = (7 << 42) | (5 << 21) | 123
    _lib.lib.nnk_status_decode(ctypes.c_uint64((~key) & 0xFFFFFFFFFFFFFFFF), ctypes.byref(st))
    assert (st.code, st.utt, st.chain, st.frame) == (1, 7, 5, 123)


def test_window_validation_matches_reference_asserts():
    import numpy as np
    from nnmnkwii_b200 import _lib
    with pytest.raises(AssertionError):  # len(coeff) != l + u + 1, paramgen/_mlpg.py:45
        _lib.make_windows([(1, 1, np.array([1.0, 2.0]))])
    with pytest.raises(NotImplementedError):
        _lib.make_windows([(0, 0, np.array([1.0]))] * 9)


def test_product_never_touches_the_oracle_or_a_cpu_fallback():
    pkg = os.path.join(ROOT, "nnmnkwii_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, re.M), f
                assert "nnk_oracle" not in src and "oracle/_ref" not in src, f
                assert "/root/reference" not in src, f


def test_cuda_sources_target_sm90a_only():
    from nnmnkwii_b200 import build
    assert "arch=compute_90a,code=sm_90a" in build.NVCC_FLAGS
    assert not any("sm_100" in f or "sm_80" in f for f in build.NVCC_FLAGS)


def test_no_gpu_means_loud_failure():
    import numpy as np
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from nnmnkwii_b200 import paramgen as G
    with pytest.raises(Exception) as ei:
        G.mlpg(np.zeros((4, 3), np.float32), np.ones((4, 3), np.float32), [(0, 0, np.array([1.0]))])
    assert "CUDA" in str(ei.value) or "cuda" in str(ei.value)


def test_host_helpers_match_reference_semantics(golden):
    import numpy as np
    from conftest import windows_set
    from nnmnkwii_b200 import paramgen as G
    # reshape_means: tests/test_paramgen.py:98-110
    m = np.random.rand(7, 6)
    r = G.reshape_means(m, 2)
    assert r.shape == (21, 2) and np.array_equal(G.reshape_means(r, 2), r)
    assert np.array_equal(r, m.reshape(7, 3, 2).transpose(1, 0, 2).reshape(-1, 2))
    # build_win_mats / full_window_mat: tests/test_paramgen.py:62-79
    for ws in windows_set():
        wm = G.build_win_mats(ws, 6)
        full = G.full_window_mat(wm, 6)
        assert full.shape == (6 * len(ws), 6)
        for i, (l, u, c) in enumerate(ws):
            blk = full[6 * i:6 * (i + 1)]
            for t in range(6):
                for k in range(-l, u + 1):
                    if 0 <= t + k < 6:
                        assert blk[t, t + k] == c[l + k]
            assert wm[i].l == l and wm[i].u == u and wm[i].transposed


def test_build_recompiles_every_object_when_the_flags_change(tmp_path, monkeypatch):
    """A changed architecture / NNK_NVCC_EXTRA must not leave objects built with the old flags behind."""
    import sys
    from nnmnkwii_b200 import build
    fake = tmp_path / "nvcc"  # records its arguments into whatever it is asked to write
    fake.write_text("#!%s\nimport sys\nopen(sys.argv[sys.argv.index('-o') + 1], 'w').write(' '.join(sys.argv[1:]))\n"
                    % sys.executable)
    fake.chmod(0o755)
    monkeypatch.setenv("NVCC", str(fake))
    monkeypatch.setattr(build, "OBJ", str(tmp_path / "obj"))
    monkeypatch.setattr(build, "LIB", str(tmp_path / "lib.so"))
    objs = [tmp_path / "obj" / s.replace(".cu", ".o") for s in build.SOURCES]
    build.build()
    first = {o: o.stat().st_mtime_ns for o in objs}
    build.build()  # nothing changed: nothing is recompiled
    assert {o: o.stat().st_mtime_ns for o in objs} == first
    monkeypatch.setattr(build, "NVCC_FLAGS", build.NVCC_FLAGS + ["-DNNK_TEST_FLAG"])
    build.build()
    for o in objs:
        assert "-DNNK_TEST_FLAG" in o.read_text(), o
