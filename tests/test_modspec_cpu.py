"""Without a GPU: the modulation-spectrum entry points refuse bad input with a clear error before touching the
device."""
import numpy as np
import pytest


def test_input_errors():
    import torch

    from nnmnkwii_b200 import preprocessing as P
    x = np.zeros((10, 2))
    with pytest.raises(ValueError, match="n must be one of"):
        P.modspec(x, n=100)
    with pytest.raises(ValueError, match="n must be one of"):
        P.modspec(x, n=8192)
    with pytest.raises(ValueError, match="n must be one of"):
        P.modspec_smoothing(x, 200, n=16)
    with pytest.raises(ValueError, match="n must be one of"):
        P.inv_modspec(np.zeros((9, 2)), np.ones((9, 2)))  # n = 16
    with pytest.raises(ValueError, match="shorter than the 300 frames"):
        P.modspec(np.zeros((300, 2)), n=256)
    with pytest.raises(RuntimeError, match="must be larger than time length"):
        P.modspec_smoothing(np.zeros((300, 2)), 200, n=256)
    with pytest.raises(ValueError, match="shorter than the 300 frames"):
        P.modspec(np.zeros((2, 400, 2)), n=256, lengths=[300, 10])
    with pytest.raises(ValueError, match="CPU tensor"):
        P.modspec(torch.zeros(10, 2))
    with pytest.raises(ValueError, match="CPU tensor"):
        P.modspec_smoothing(torch.zeros(10, 2), 200)
    with pytest.raises(ValueError, match="CPU tensor"):
        P.inv_modspec(np.zeros((129, 2)), torch.ones(129, 2))
    with pytest.raises(TypeError, match="float32 or float64"):
        P.modspec(np.zeros((10, 2), np.int64))
    with pytest.raises(TypeError, match="float32 or float64"):
        P.modspec_smoothing(np.zeros((10, 2), np.float16), 200)
    with pytest.raises(TypeError, match="CUDA tensor or a NumPy array"):
        P.modspec([[0.0, 1.0]])
    with pytest.raises(ValueError, match="Invalid norm"):
        P.modspec(x, n=256, norm="unitary")
    with pytest.raises(ValueError, match="Nyquist"):
        P.modspec_smoothing(x, 200, n=256, cutoff=101)
    with pytest.raises(ValueError, match="lengths exceed"):
        P.modspec(np.zeros((2, 10, 2)), n=256, lengths=[11, 3])
    with pytest.raises(ValueError, match="lengths exceed"):
        P.inv_modspec(np.zeros((2, 129, 2)), np.ones((2, 129, 2)), lengths=[257, 3])
    with pytest.raises(ValueError, match="lengths has 1 entries"):
        P.modspec(np.zeros((2, 10, 2)), n=256, lengths=[3])
    with pytest.raises(ValueError, match="padded"):
        P.modspec(x, n=256, lengths=[10])
    with pytest.raises(ValueError, match="differ in shape"):
        P.inv_modspec(np.zeros((129, 2)), np.ones((129, 3)))
    with pytest.raises(ValueError, match=r"\(T, D\) or \(B, T, D\)"):
        P.modspec(np.zeros(10), n=256)

