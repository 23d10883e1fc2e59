"""Write wave_reference_golden.npz from the reference built under oracle/_ref/ (data only).

    python tests/golden/make_wave_golden.py

Needs the reference package in oracle/_ref (oracle/build_ref.sh) and its example data.  Stores
  * ``audio``: AUDIO_LEN samples of example_audio_file() from AUDIO_START (int16, speech);
  * ``lf0_<i>``: raw log-F0 of the three example acoustic utterances, Y_acoustic[:, 180] *
    Y_acoustic[:, 183] (lf0 masked by vuv: the unvoiced pattern of real speech), float32;
  * the reference's outputs on them:
      - interp1d for every two-point kind on (T,) float32 / float64 inputs (values), and on (T, 1)
        inputs as digests;
      - preemphasis / inv_preemphasis for coef in COEFS on the audio scaled to [-1, 1) in float32 and
        float64, as SHA-256 digests (the functions must be bit-identical; a digest says so in 64 bytes);
      - the mu-law family for mu in MUS on the first MU_LEN samples (values, with their dtypes);
      - adjust_frame_length(s) on crafted shapes, with np.pad keyword arguments.
Every input is deterministic, so two runs write identical arrays.
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
AUDIO_START, AUDIO_LEN, MU_LEN = 8000, 16000, 1024
KINDS = ("linear", "slinear", "zero", "nearest", "nearest-up", "previous", "next")
COEFS = (0.97, 0.86, 0.0)
MUS = (256, 2)


def digest(a):
    """'dtype shape sha256' of an array's C-order bytes."""
    a = np.ascontiguousarray(a)
    return np.array("%s %s %s" % (a.dtype.str, "x".join(map(str, a.shape)), hashlib.sha256(a.tobytes()).hexdigest()))


def adjust_cases():
    """(name, x, y or None, kwargs) of the adjust_frame_length(s) checks."""
    r = np.random.RandomState(0)
    a1, a2 = r.randn(10, 3), r.randn(13, 3)
    v1, v2 = r.randn(7), r.randn(9)
    return [
        ("one_pad3", a1, None, dict(pad=True, divisible_by=3)),
        ("one_trim3", a1, None, dict(pad=False, divisible_by=3)),
        ("one_same", a1, None, dict(divisible_by=5)),
        ("one_vec_edge", v1, None, dict(divisible_by=4, mode="edge")),
        ("one_const7", a1, None, dict(divisible_by=4, constant_values=7.0)),
        ("two_pad", a1, a2, dict()),
        ("two_trim", a1, a2, dict(pad=False)),
        ("two_even", a1, a2, dict(ensure_even=True)),
        ("two_pad4_reflect", a1, a2, dict(divisible_by=4, mode="reflect")),
        ("two_trim4", a1, a2, dict(pad=False, divisible_by=4)),
        ("two_vec", v1, v2, dict(divisible_by=2, mode="edge")),
    ]


def main():
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    from scipy.io import wavfile

    from nnmnkwii import preprocessing as P
    from nnmnkwii.datasets import FileSourceDataset
    from nnmnkwii.util import example_audio_file, example_file_data_sources_for_acoustic_model
    out = {}
    _, audio = wavfile.read(example_audio_file())
    audio = audio[AUDIO_START:AUDIO_START + AUDIO_LEN].astype(np.int16)
    out["audio"] = audio
    _, Ys = example_file_data_sources_for_acoustic_model()
    Y = FileSourceDataset(Ys)
    for i in range(3):
        lf0 = (Y[i][:, 180] * Y[i][:, 183]).astype(np.float32)
        out["lf0_%d" % i] = lf0
        for dt in (np.float32, np.float64):
            for kind in KINDS:
                key = "interp_%d_%s_%s" % (i, np.dtype(dt).name, kind)
                out[key] = P.interp1d(lf0.astype(dt), kind=kind)
                out[key + "_col"] = digest(P.interp1d(lf0.astype(dt)[:, None], kind=kind))
    for dt in (np.float32, np.float64):
        x = (audio / 32768.0).astype(dt)
        for c in COEFS:
            out["pre_%s_%g" % (np.dtype(dt).name, c)] = digest(P.preemphasis(x, coef=c))
            out["inv_%s_%g" % (np.dtype(dt).name, c)] = digest(P.inv_preemphasis(x, coef=c))
    for mu in MUS:
        for dt in (np.float32, np.float64):
            x = (audio[:MU_LEN] / 32768.0).astype(dt)
            tag = "%d_%s" % (mu, np.dtype(dt).name)
            y = P.mulaw(x, mu)
            q = P.mulaw_quantize(x, mu)
            iy = P.inv_mulaw(y.astype(dt), mu)
            iq = P.inv_mulaw_quantize(q, mu)
            for name, v in (("mulaw", y), ("quant", q), ("inv", iy), ("invq", iq)):
                out["mu_%s_%s" % (name, tag)] = v
                out["mu_%s_%s_dtype" % (name, tag)] = np.array(v.dtype.str)
    for name, x, y, kw in adjust_cases():
        if y is None:
            out["adj_" + name] = P.adjust_frame_length(x, **kw)
        else:
            out["adj_%s_x" % name], out["adj_%s_y" % name] = P.adjust_frame_lengths(x, y, **kw)
    np.savez_compressed(os.path.join(HERE, "wave_reference_golden.npz"), **out)


if __name__ == "__main__":
    main()
