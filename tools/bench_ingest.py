"""Time the reference's per-clip transform -- Resize(256, antialias=True) -> CenterCrop(256) -> Normalize(.5, .5) of
frames/255 -- on one 17 x 1080 x 1920 x 3 uint8 clip, three ways:

  kernel       vidtok_b200.video_io.transform_frames (one launch), CUDA events
  cpu          the reference's torchvision transform on the host CPU (the DataLoader path), wall clock
  torch_gpu    torch.nn.functional.interpolate(antialias=True) on the GPU, then the crop and the Normalize, CUDA events

and the kernel's achieved bytes/s (algorithmic bytes from the library profiler: the source rectangle under the crop's
taps, read once, plus the fp32 clip written once) against the H100 SXM data-sheet 3.35 TB/s.  Prints one JSON line with
the card, its power limit and SM clocks.
usage: python tools/bench_ingest.py [--iters 50] [--cpu-iters 5] [--out FILE]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vidtok_b200 import _native as N  # noqa: E402
from vidtok_b200.video_io import resize_crop_geometry, transform_frames  # noqa: E402

T, HS, WS, CH, SIZE = 17, 1080, 1920, 3, 256
PEAK_BPS = 3.35e12


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[torch.cuda.current_device()]
    except Exception as e:    # the numbers are still printed, without the card's settings
        return f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {e})"


def gpu_ms(fn, iters):
    for _ in range(5):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--cpu-iters", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ingest: no CUDA device; the kernel numbers need an H100")

    g = torch.Generator().manual_seed(0)
    host = torch.randint(0, 256, (T, HS, WS, CH), generator=g, dtype=torch.uint8)
    dev = host.cuda()
    Hr, Wr, h0, w0 = resize_crop_geometry(HS, WS, SIZE, SIZE)

    def kernel():
        return transform_frames(dev, SIZE, SIZE)

    def torch_gpu():
        x = F.interpolate(dev.permute(0, 3, 1, 2).float() / 255.0, size=(Hr, Wr), mode="bilinear", align_corners=False,
                          antialias=True)
        return ((x[:, :, h0:h0 + SIZE, w0:w0 + SIZE] - 0.5) / 0.5).permute(1, 0, 2, 3)

    before = card()
    k_ms = gpu_ms(kernel, args.iters)
    t_ms = gpu_ms(torch_gpu, args.iters)
    k_ms2 = gpu_ms(kernel, args.iters)       # again, after the torch path: the spread of the kernel's own time
    lib = N.lib()
    buf = C.create_string_buffer(1 << 14)
    lib.vt_profile_start()
    kernel()
    lib.vt_profile_stop(buf, len(buf))
    nbytes = json.loads(buf.value.decode())["u8_frames_resize_to_clip"]["bytes"]
    after = card()

    from torchvision import transforms
    tf = transforms.Compose([transforms.Resize(SIZE, antialias=True), transforms.CenterCrop((SIZE, SIZE)),
                             transforms.Normalize(mean=(0.5,) * 3, std=(0.5,) * 3)])

    def cpu():
        return tf(host.permute(0, 3, 1, 2).float() / 255.0).permute(1, 0, 2, 3)
    cpu()
    t0 = time.perf_counter()
    for _ in range(args.cpu_iters):
        cpu()
    c_ms = (time.perf_counter() - t0) * 1e3 / args.cpu_iters

    k_best = min(k_ms, k_ms2)
    res = {
        "clip": f"{T}x{HS}x{WS}x{CH} uint8 -> {CH}x{T}x{SIZE}x{SIZE} fp32 (resize to {Hr}x{Wr})",
        "card_before": before, "card_after": after,
        "kernel_ms": [round(k_ms, 4), round(k_ms2, 4)],
        "kernel_frames_per_s": round(T / k_best * 1e3, 1),
        "kernel_bytes": nbytes,
        "kernel_TBps": round(nbytes / (k_best * 1e-3) / 1e12, 3),
        "kernel_share_of_3.35TBps": round(nbytes / (k_best * 1e-3) / PEAK_BPS, 3),
        "torch_gpu_ms": round(t_ms, 4),
        "cpu_ms": round(c_ms, 2), "cpu_threads": torch.get_num_threads(), "cpu_count": os.cpu_count(),
        "cpu_frames_per_s": round(T / c_ms * 1e3, 1),
    }
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
