"""Time corpus normalisation (csrc/nnk_stats.cu) at two scales.

    python tools/bench_normalize.py [--iters 20] [--host-utts 1024] [--ref-utts 512]

187 columns, float32, T drawn as bench.py draws them:
  cfg1: 256 utterances of T ~ U{540..660} (about 1.5e5 frames);
  cfg4: 8192 utterances of T ~ U{200..2000} (about 9.0e6 frames, 6.7 GB of valid frames).
Per scale, on a padded (B, Tmax, 187) CUDA tensor with lengths, after a warm-up, median of CUDA events:
  * `nnk_frame_stats` alone and the whole `meanvar` call: ms, GB/s of valid bytes, share of the H100 SXM
    data-sheet 3.35 TB/s;
  * `scale` over the whole padded tensor: ms and GB/s of bytes read plus written.
Form (a), a list of host NumPy arrays, is timed on the first --host-utts utterances; it streams through
page-locked staging and is bound by host packing and host-to-device copies, so it is reported as such.
The restated reference loop (oracle/normalize.py: scikit-learn's _incremental_mean_and_var per utterance)
runs on the host over the first --ref-utts cfg4 utterances.  The card name and power limit are read in
the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_BW = 3.35e12
D = 187


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        idx = os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0] or "0"
        out = subprocess.run(["nvidia-smi", "-i", idx, "--query-gpu=power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        out = "unknown (%s)" % type(e).__name__
    return name, out


def lengths():
    return {"cfg1": np.random.default_rng(1234).integers(540, 661, size=256),
            "cfg4": np.random.default_rng(4242).integers(200, 2001, size=8192)}


def events(fn, reps):
    import torch
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def device_runs(name, lens, iters, gpu, power):
    import torch

    from nnmnkwii_b200 import _device as dev
    from nnmnkwii_b200 import _lib
    from nnmnkwii_b200 import preprocessing as P
    B, Tmax = len(lens), int(lens.max())
    frames = int(lens.sum())
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn((B, Tmax, D), generator=g, device="cuda", dtype=torch.float32)
    valid = frames * D * 4
    st = dev.current_stream_ptr(x.device)
    state = torch.zeros(1 + 4 * D, dtype=torch.float64, device="cuda")
    off = torch.arange(B + 1, dtype=torch.int64, device="cuda") * Tmax
    l32 = torch.as_tensor(lens.astype(np.int32), device="cuda")
    ws = torch.empty(int(_lib.lib.nnk_frame_stats_workspace_bytes(B, Tmax, D)), dtype=torch.uint8, device="cuda")

    def kernel():
        _lib.check(_lib.lib.nnk_frame_stats(x.data_ptr(), _lib.NNK_F32, D, D, off.data_ptr(), l32.data_ptr(), B, Tmax,
                                            state.data_ptr(), ws.data_ptr(), ws.numel(), st), "stats")

    m, v = P.meanvar(x, lens)
    s = torch.sqrt(v)
    for _ in range(3):
        kernel()
        P.meanvar(x, lens)
        P.scale(x, m, s)
    torch.cuda.synchronize()
    k_ms = events(kernel, iters)
    mv_ms = events(lambda: P.meanvar(x, lens), iters)
    sc_ms = events(lambda: P.scale(x, m, s), max(3, iters // 2))
    for what, ms in (("frame_stats_kernel", k_ms), ("meanvar_call", mv_ms)):
        print(json.dumps({"workload": name, "op": what, "form": "padded CUDA tensor", "utterances": B, "frames": frames,
                          "D": D, "dtype": "float32", "ms": round(ms, 4), "valid_GB_per_s": valid / (ms * 1e-3) / 1e9,
                          "share_of_3.35TB_s": valid / (ms * 1e-3) / PEAK_BW, "gpu": gpu, "power_limit": power}))
    moved = 2 * x.numel() * 4
    print(json.dumps({"workload": name, "op": "scale", "form": "padded CUDA tensor (every frame)", "elements": x.numel(),
                      "ms": round(sc_ms, 4), "GB_per_s_read_plus_write": moved / (sc_ms * 1e-3) / 1e9,
                      "share_of_3.35TB_s": moved / (sc_ms * 1e-3) / PEAK_BW, "gpu": gpu, "power_limit": power}))
    del x
    torch.cuda.empty_cache()


def host_runs(name, lens, gpu, power):
    from nnmnkwii_b200 import preprocessing as P
    rng = np.random.default_rng(7)
    utts = [rng.standard_normal((int(t), D), dtype=np.float32) for t in lens]
    P.meanvar(utts[:8])
    t0 = time.perf_counter()
    P.meanvar(utts)
    dt = time.perf_counter() - t0
    frames = int(lens.sum())
    print(json.dumps({"workload": name, "op": "meanvar", "form": "list of host arrays (bound by host packing and "
                      "host-to-device copies)", "utterances": len(lens), "frames": frames, "ms": round(dt * 1e3, 3),
                      "host_GB_per_s": frames * D * 4 / dt / 1e9, "gpu": gpu, "power_limit": power}))


def reference_loop(lens):
    from oracle import normalize as R
    rng = np.random.default_rng(8)
    utts = [rng.standard_normal((int(t), D), dtype=np.float32) for t in lens]
    t0 = time.perf_counter()
    R.meanvar(utts)
    dt = time.perf_counter() - t0
    frames = int(lens.sum())
    print(json.dumps({"op": "meanvar", "form": "restated reference loop on the host (oracle/normalize.py, "
                      "scikit-learn per utterance)", "utterances": len(lens), "frames": frames,
                      "seconds": round(dt, 3), "frames_per_s": frames / dt}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--host-utts", type=int, default=1024)
    ap.add_argument("--ref-utts", type=int, default=512)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_normalize: no CUDA device (these are GPU timings; there is no CPU fallback)")
    torch.cuda.set_device(0)
    gpu, power = card()
    L = lengths()
    for name in ("cfg1", "cfg4"):
        device_runs(name, L[name], args.iters, gpu, power)
    host_runs("cfg1", L["cfg1"], gpu, power)
    host_runs("cfg4[:%d]" % args.host_utts, L["cfg4"][:args.host_utts], gpu, power)
    reference_loop(L["cfg4"][:args.ref_utts])


if __name__ == "__main__":
    main()
