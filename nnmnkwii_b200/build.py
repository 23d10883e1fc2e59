"""Build libnnk_b200.so (sm_90a only: H100) in-tree with nvcc.

    python -m nnmnkwii_b200.build [--force]

The library is the product: every numeric entry point of the package calls into it through the C
ABI declared in include/nnk_b200.h.  There is no fallback if it is missing.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "csrc", "_obj")
LIB = os.environ.get("NNK_LIB_OUT") or os.path.join(HERE, "libnnk_b200.so")  # NNK_LIB_OUT: A/B builds
SOURCES = ["nnk_core.cu", "nnk_mlpg.cu", "nnk_host.cu", "nnk_uvmlpg.cu", "nnk_dtw.cu", "nnk_delta.cu", "nnk_metrics.cu", "nnk_shard.cu", "nnk_gmm.cu",
           "nnk_gmm_em.cu", "nnk_kmeans.cu", "nnk_postfilter.cu", "nnk_stats.cu", "nnk_wave.cu", "nnk_linalg.cu",
           "nnk_modspec.cu", "nnk_gmm_traj.cu", "nnk_ms_segment.cu", "nnk_ms_gen.cu", "nnk_mix_gen.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
] + os.environ.get("NNK_NVCC_EXTRA", "").split()  # e.g. -DNNK_EXP_WS_F32 for A/B experiments


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def _newer(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    # objects built with other flags (architecture, NNK_NVCC_EXTRA) or another nvcc are stale whatever their age
    stamp = os.path.join(OBJ, "flags.txt")
    flags = " ".join([_nvcc()] + NVCC_FLAGS)
    if not os.path.exists(stamp) or open(stamp).read() != flags:
        force = True
    srcs = [s for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    include = os.path.join(os.path.dirname(HERE), "include")
    headers += [os.path.join(include, f) for f in os.listdir(include) if f.endswith(".h")]
    jobs = []
    objs = []
    for s in srcs:
        src = os.path.join(CSRC, s)
        obj = os.path.join(OBJ, s.replace(".cu", ".o"))
        objs.append(obj)
        if force or _newer(obj, [src] + headers):
            jobs.append([_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj])
    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            for cmd, res in zip(jobs, ex.map(lambda c: subprocess.run(c, capture_output=True, text=True), jobs)):
                if verbose or res.returncode:
                    sys.stderr.write(res.stdout + res.stderr)
                if res.returncode:
                    raise RuntimeError("nvcc failed: " + " ".join(cmd))
        with open(stamp, "w") as f:
            f.write(flags)
    if jobs or force or _newer(LIB, objs):
        cmd = [_nvcc(), "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB] + objs
        subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
