"""Corpus normalisation oracle: a restatement of the reference's loops, not the reference.
TEST INFRASTRUCTURE, NOT PRODUCT.

``meanvar`` restates nnmnkwii/preprocessing/generic.py:496-549 literally: per utterance (cut to
``lengths[idx]``), scikit-learn's ``_incremental_mean_and_var``, then a cast to ``dataset[0].dtype``.
``minmax`` restates :605-636 (``np.minimum`` / ``np.maximum`` per utterance).  The scaling functions are
the reference's NumPy expressions.  tests/golden/normalize_reference_golden.npz holds the reference's own
outputs; tests/test_normalize_cpu.py checks that this restatement reproduces them.
"""
import numpy as np
from sklearn.utils.extmath import _incremental_mean_and_var

__all__ = ["meanvar", "meanstd", "minmax", "scale", "inv_scale", "minmax_scale_params", "minmax_scale",
           "inv_minmax_scale"]


def _handle_zeros_in_scale(scale):
    if np.isscalar(scale):
        return 1.0 if scale == 0.0 else scale
    scale = scale.copy()
    scale[scale == 0.0] = 1.0
    return scale


def meanvar(dataset, lengths=None, mean_=0.0, var_=0.0, last_sample_count=0, return_last_sample_count=False):
    dtype = dataset[0].dtype
    for idx, x in enumerate(dataset):
        if lengths is not None:
            x = x[: lengths[idx]]
        mean_, var_, _ = _incremental_mean_and_var(x, mean_, var_, last_sample_count)
        last_sample_count += len(x)
    mean_, var_ = mean_.astype(dtype), var_.astype(dtype)
    if return_last_sample_count:
        return mean_, var_, last_sample_count
    return mean_, var_


def meanstd(dataset, lengths=None, mean_=0.0, var_=0.0, last_sample_count=0, return_last_sample_count=False):
    ret = meanvar(dataset, lengths, mean_, var_, last_sample_count, return_last_sample_count)
    s = _handle_zeros_in_scale(np.sqrt(ret[1]))
    return (ret[0], s) + tuple(ret[2:])


def minmax(dataset, lengths=None):
    max_ = -np.inf
    min_ = np.inf
    for idx, x in enumerate(dataset):
        if lengths is not None:
            x = x[: lengths[idx]]
        min_ = np.minimum(min_, np.min(x, axis=(0,)))
        max_ = np.maximum(max_, np.max(x, axis=(0,)))
    return min_, max_


def scale(x, data_mean, data_std):
    return (x - data_mean) / _handle_zeros_in_scale(data_std)


def inv_scale(x, data_mean, data_std):
    return data_std * x + data_mean


def _factor(data_min, data_max, feature_range):
    return (feature_range[1] - feature_range[0]) / _handle_zeros_in_scale(data_max - data_min)


def minmax_scale_params(data_min, data_max, feature_range=(0, 1)):
    scale_ = _factor(data_min, data_max, feature_range)
    return feature_range[0] - data_min * scale_, scale_


def minmax_scale(x, data_min=None, data_max=None, feature_range=(0, 1), scale_=None, min_=None):
    if scale_ is None:
        scale_ = _factor(data_min, data_max, feature_range)
    if min_ is None:
        min_ = feature_range[0] - data_min * scale_
    return x * scale_ + min_


def inv_minmax_scale(x, data_min=None, data_max=None, feature_range=(0, 1), scale_=None, min_=None):
    if scale_ is None:
        scale_ = _factor(data_min, data_max, feature_range)
    if min_ is None:
        min_ = feature_range[0] - data_min * scale_
    return (x - min_) / scale_
