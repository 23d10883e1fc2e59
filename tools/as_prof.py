"""Phase timers of mlpg_fwd_as_kernel: per-CTA clock64 cycles of every assembler and solver phase on the three
MLPG workloads the benchmark reports (configs[1], T=1000 forward, T=1000 gradient).  Needs a library built with
the counters, e.g. next to the normal one:

    NNK_NVCC_EXTRA=-DNNK_AS_PROF NNK_LIB_OUT=/tmp/libnnk_prof.so python -m nnmnkwii_b200.build
    NNK_LIB_PATH=/tmp/libnnk_prof.so python tools/as_prof.py

(the build stamps its flags, so the next plain build recompiles every object)."""
import ctypes
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from nnmnkwii_b200 import _device as dev, _lib, paramgen as G  # noqa: E402

if not hasattr(_lib.lib, "nnk_as_prof_read"):
    sys.exit("%s was built without -DNNK_AS_PROF" % _lib.LIB_PATH)
device = torch.device("cuda", 0)
wc = _lib.make_windows(bench.WINDOWS)

# configs[1]: the benchmark's batch (Merlin layout, 63 chains = 2 groups per utterance)
lens, means, variances = bench.make_batch(0)
layout = G.merlin_layout()
off = torch.from_numpy(np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)).to(device)
d_m, d_v = torch.from_numpy(means).to(device), torch.from_numpy(variances).to(device)
d_out = torch.zeros((int(lens.sum()), 63), dtype=torch.float32, device=device)
order = torch.from_numpy(np.argsort(-lens, kind="stable").astype(np.int32)).to(device)
chains = dev.chains_on_device(layout.chains, device)


def cfg2():
    dev.run_mlpg("fwd", means=d_m, variances=d_v, rhs=None, out=d_out, offsets=off, lengths=None, order=order,
                 chains=chains, n_chain=layout.n_chain, max_T=int(lens.max()), windows_c=wc, in_ld=187, var_ld=187,
                 go_ld=0, out_ld=63, dtype_code=_lib.NNK_F32, go_f64=0, n_utt=len(lens), device=device, check=False)


# the T=1000 shapes of bench.bench_extras: 256 utterances, static_dim 60, per-frame variances
B2, T2, sd2 = 256, 1000, 60
g = torch.Generator(device=device).manual_seed(0)
ch2 = dev.chains_on_device(dev.simple_chains(sd2), device)
off2 = torch.arange(B2 + 1, dtype=torch.int64, device=device) * T2
m2 = torch.rand(B2 * T2, 3 * sd2, device=device, generator=g)
v2 = torch.rand(B2 * T2, 3 * sd2, device=device, generator=g) + 0.1
go2 = torch.randn(B2 * T2, sd2, device=device, generator=g)
y2 = torch.zeros(B2 * T2, sd2, device=device)
g2 = torch.zeros(B2 * T2, 3 * sd2, device=device)


def t1000(mode, rhs, o, out_ld):
    dev.run_mlpg(mode, means=m2, variances=v2, rhs=rhs, out=o, offsets=off2, lengths=None, order=None, chains=ch2,
                 n_chain=sd2, max_T=T2, windows_c=wc, in_ld=3 * sd2, var_ld=3 * sd2, go_ld=sd2, out_ld=out_ld,
                 dtype_code=_lib.NNK_F32, go_f64=0, n_utt=B2, device=device, check=False)


cases = (("configs[1]", cfg2), ("T1000 forward", lambda: t1000("fwd", None, y2, sd2)),
         ("T1000 gradient", lambda: t1000("grad", go2, g2, 3 * sd2)))
# forward pass phases, then the whole backward pass (forward solves: the segment replay; assemblers
# >= AS_NA_B only wait at the pass boundary).  Solver: forward pass, then backward: forward solves wait for
# replayed band rows / replay + back-substitute (waits included); gradients wait for scratch TMA / backward
A_PH = ["wait pb_empty", "wait input TMA", "convert+assemble+publish", "replay pass (fwd solves)"]
S_PH = ["wait pb_full", "eliminate", "wait replay rows | scratch TMA", "replay+backward | backward"]
SLOTS = 40  # NNK_AS_PROF_SLOTS: [role * 4 + phase], [32] CTAs, [33] G, [34] NA
buf = (ctypes.c_ulonglong * SLOTS)()
print("%s, per-CTA average cycles of each warp (assembler q.h: tile ownership q of chain group h of the CTA)"
      % torch.cuda.get_device_name(0))
for title, fn in cases:
    for _ in range(3):
        fn()
    _lib.lib.nnk_as_prof_read(buf)  # synchronises and clears the counters
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    _lib.lib.nnk_as_prof_read(buf)
    n_cta, G, na = int(buf[32]), int(buf[33]), int(buf[34])
    print("%s: G = %d, NA = %d, %d CTAs, launch %.3f ms (instrumented)" % (title, G, na, n_cta, e0.elapsed_time(e1)))
    for i, ph in enumerate(A_PH):
        per = [buf[(h * na + q) * 4 + i] / n_cta for h in range(G) for q in range(na)]
        print("  A %-26s" % ph + "".join("%10.0f" % x for x in per) + "   mean %.0f" % (sum(per) / len(per)))
    for i, ph in enumerate(S_PH):
        per = [buf[(G * na + h) * 4 + i] / n_cta for h in range(G)]
        print("  S %-26s" % ph + "".join("%10.0f" % x for x in per))
