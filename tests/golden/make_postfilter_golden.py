"""Write merlin_post_filter_golden.npz from the reference's test data (data only, no code is copied).

Run where a checkout of the reference (r9y9/nnmnkwii v0.1.3) exists:

    python tests/golden/make_postfilter_golden.py [REFERENCE_DIR]

REFERENCE_DIR defaults to $NNK_REFERENCE_DIR, else /root/reference (the same default as
oracle/build_ref.sh).  The reference's tests/data/merlin_post_filter/ holds Merlin's SPTK command-line
output for arctic_b0539 (525 frames x 60 coefficients, float32): the input, the weight file and every
intermediate of the post-filter chain.  tests/test_postfilter_cpu.py, tests/test_postfilter_gpu.py and
__graft_entry__.smoke() compare against the arrays this writes.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def main(ref_dir=None):
    ref_dir = ref_dir or os.environ.get("NNK_REFERENCE_DIR", "/root/reference")
    src = os.path.join(ref_dir, "tests", "data", "merlin_post_filter")
    out = {"weight": np.fromfile(os.path.join(src, "weight"), dtype=np.float32)}
    for name in ("mgc", "mgc_r0", "mgc_p_r0", "mgc_b0", "mgc_p_b0", "mgc_p_mgc"):
        a = np.fromfile(os.path.join(src, "arctic_b0539." + name), dtype=np.float32)
        out[name] = a.reshape(-1, 60) if name in ("mgc", "mgc_p_mgc") else a
    np.savez_compressed(os.path.join(HERE, "merlin_post_filter_golden.npz"), **out)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else None)
