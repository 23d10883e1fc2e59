"""Write normalize_reference_golden.npz from the reference built under oracle/_ref/ (data only).

    python tests/golden/make_normalize_golden.py

Needs the reference package in oracle/_ref (oracle/build_ref.sh) and its example data: the three
slt_arctic_demo_data utterances, X_acoustic (425 columns) and Y_acoustic (187 columns), float32.  To keep
the file small, the inputs are a window of each utterance (frames 150 .. 150 + WINDOW[i]: speech, not the
leading silence) rather than all ~600 frames.  Stores those inputs, and the reference's own outputs of
  * meanvar / meanstd / minmax, plain and padded to 1000 frames with lengths;
  * the incremental split of the reference's test_meanvar_incremental (its input is regenerated from
    np.random.seed(1234), as that test does, so only the outputs are stored);
  * scale / inv_scale / minmax_scale / inv_minmax_scale on utterance 0, as SHA-256 digests of the result
    bytes (with shape and dtype): the functions must be bit-identical, and a digest says so in 64 bytes;
  * minmax_scale_params, and remove_zeros_frames on a crafted matrix.
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
START, WINDOW = 150, (64, 96, 72)


def digest(a):
    """'dtype shape sha256' of an array's C-order bytes."""
    a = np.ascontiguousarray(a)
    return np.array("%s %s %s" % (a.dtype.str, "x".join(map(str, a.shape)), hashlib.sha256(a.tobytes()).hexdigest()))


def main():
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    from nnmnkwii import preprocessing as P
    from nnmnkwii.util import example_file_data_sources_for_acoustic_model
    from nnmnkwii.datasets import FileSourceDataset
    Xs, Ys = example_file_data_sources_for_acoustic_model()
    X = [x[START:START + w] for x, w in zip(FileSourceDataset(Xs), WINDOW)]
    Y = [y[START:START + w] for y, w in zip(FileSourceDataset(Ys), WINDOW)]
    out = {}
    for name, data in (("X", X), ("Y", Y)):
        lengths = np.array([len(u) for u in data])
        out[name + "_lengths"] = lengths
        for i, u in enumerate(data):
            out["%s_%d" % (name, i)] = u
        pad = np.zeros((len(data), 1000, data[0].shape[1]), dtype=data[0].dtype)
        for i, u in enumerate(data):
            pad[i, :len(u)] = u
        out[name + "_mean"], out[name + "_var"] = P.meanvar(data)
        _, out[name + "_std"] = P.meanstd(data)
        out[name + "_min"], out[name + "_max"] = P.minmax(data)
        out[name + "_pad_mean"], out[name + "_pad_var"] = P.meanvar(pad, lengths)
        _, out[name + "_pad_std"] = P.meanstd(pad, lengths)
        out[name + "_pad_min"], out[name + "_pad_max"] = P.minmax(pad, lengths)
    # scaling on utterance 0: scale family on Y, min/max family on X (the TTS notebook's use)
    y0, x0 = Y[0], X[0]
    sy = P.scale(y0, out["Y_mean"], out["Y_std"].copy())
    sx = P.minmax_scale(x0, out["X_min"], out["X_max"], feature_range=(0.01, 0.99))
    out["scale_Y0"] = digest(sy)
    out["inv_scale_Y0"] = digest(P.inv_scale(sy, out["Y_mean"], out["Y_std"]))
    out["minmax_scale_X0"] = digest(sx)
    out["inv_minmax_scale_X0"] = digest(P.inv_minmax_scale(sx, out["X_min"], out["X_max"], feature_range=(0.01, 0.99)))
    out["params_min_"], out["params_scale_"] = P.minmax_scale_params(out["X_min"], out["X_max"],
                                                                     feature_range=(0.01, 0.99))
    # the incremental split of the reference's test_meanvar_incremental
    np.random.seed(1234)
    inc = np.random.randn(32, 100, 24)
    out["inc_mean_a"], out["inc_var_a"], out["inc_count_a"] = P.meanvar(inc[:16], return_last_sample_count=True)
    out["inc_mean_b"], out["inc_var_b"] = P.meanvar(inc[16:], mean_=out["inc_mean_a"], var_=out["inc_var_a"],
                                                    last_sample_count=out["inc_count_a"])
    out["inc_mean"], out["inc_var"] = P.meanvar(inc)
    # remove_zeros_frames on a crafted matrix: zero rows, rows below eps, a row exactly at eps, negatives
    rz = np.random.RandomState(0).randn(12, 5)
    rz[[0, 3, 11]] = 0.0
    rz[5] = 1e-9
    rz[7] = [2e-8, 0.0, 0.0, 0.0, 0.0]
    rz[8] = [-1e-7, 0.0, 0.0, 0.0, 0.0]
    out["rz_in"] = rz
    out["rz_out"] = P.remove_zeros_frames(rz)
    np.savez_compressed(os.path.join(HERE, "normalize_reference_golden.npz"), **out)


if __name__ == "__main__":
    main()
