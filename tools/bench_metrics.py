"""Time the evaluation protocol's PSNR + SSIM of a reconstruction (scripts/inference_evaluate.py:175-186) two ways on the
same device, for three workloads:

  fused        vidtok_b200.metrics.frame_scores: one pass over the two clips plus a small finishing kernel
  torch        what it replaces: clamp, (v + 1) / 2, compat_util.compute_psnr + compute_ssim on CUDA tensors

  kl488_fp32   8 x 3 x 17 x 256 x 256, fp32 input and reconstruction (the kl488 benchmark batch)
  kl488_bf16   the same with a bf16 reconstruction (the engine's output inside an autocast region)
  1080p        1 x 3 x 17 x 1080 x 1920 fp32 (SSIM pool factor 4)

CUDA events around warmed loops; per workload also the peak memory each path allocates beyond its inputs
(torch.cuda.max_memory_allocated) and the fused kernels' algorithmic bytes (both clips read once, from the library's
profiler) over their time against the H100 SXM data-sheet 3.35 TB/s.  Prints one JSON line with the card, its power limit
and SM clocks.
usage: python tools/bench_metrics.py [--seconds 0.5] [--out FILE]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vidtok_b200 import _native as N  # noqa: E402
from vidtok_b200.compat_util import compute_psnr, compute_ssim  # noqa: E402
from vidtok_b200.metrics import frame_scores  # noqa: E402

PEAK_BPS = 3.35e12
WORKLOADS = [("kl488_fp32", (8, 3, 17, 256, 256), torch.float32),
             ("kl488_bf16", (8, 3, 17, 256, 256), torch.bfloat16),
             ("1080p", (1, 3, 17, 1080, 1920), torch.float32)]


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[torch.cuda.current_device()]
    except Exception as e:    # the numbers are still printed, without the card's settings
        return f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {e})"


def gpu_ms(fn, seconds):
    """mean time of fn over a warmed loop sized to fill about `seconds`"""
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    iters = max(5, int(seconds * 1e3 / max(a.elapsed_time(b), 1e-3)))
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters, iters


def peak_extra_bytes(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = fn()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del out
    return peak


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=0.5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_metrics: no CUDA device; the numbers need an H100")
    lib = N.lib()
    res = {"card_before": card(), "workloads": {}}
    for name, shape, ydt in WORKLOADS:
        g = torch.Generator(device="cuda").manual_seed(0)
        x = (torch.rand(shape, generator=g, device="cuda") * 2 - 1)
        y = (x + 0.1 * torch.randn(shape, generator=g, device="cuda")).to(ydt)

        def fused():
            return frame_scores(x, y)

        def torch_chain():
            out = y.clamp(-1, 1)
            a, b = (x + 1) / 2, (out + 1) / 2
            return compute_psnr(a, b), compute_ssim(a.float(), b.float())

        f_ms, f_it = gpu_ms(fused, args.seconds)
        t_ms, t_it = gpu_ms(torch_chain, args.seconds)
        f_ms2, _ = gpu_ms(fused, args.seconds)      # again, after the torch path: the spread of the fused time
        buf = C.create_string_buffer(1 << 14)
        lib.vt_profile_start()
        fused()
        lib.vt_profile_stop(buf, len(buf))
        prof = json.loads(buf.value.decode())
        nbytes = prof["frame_scores"]["bytes"]
        best = min(f_ms, f_ms2)
        res["workloads"][name] = {
            "shape": "x".join(map(str, shape)), "y_dtype": str(ydt).replace("torch.", ""), "frames": shape[0] * shape[2],
            "fused_ms": [round(f_ms, 4), round(f_ms2, 4)], "fused_iters": f_it,
            "torch_ms": round(t_ms, 4), "torch_iters": t_it, "speedup": round(t_ms / best, 2),
            "fused_peak_MB": round(peak_extra_bytes(fused) / 1e6, 3), "torch_peak_MB": round(peak_extra_bytes(torch_chain) / 1e6, 1),
            "fused_bytes": nbytes, "fused_TBps": round(nbytes / (best * 1e-3) / 1e12, 3),
            "fused_share_of_3.35TBps": round(nbytes / (best * 1e-3) / PEAK_BPS, 3),
            "profiled_ms": {k: round(v["ms"], 4) for k, v in prof.items()},
        }
        del x, y
        torch.cuda.empty_cache()
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
