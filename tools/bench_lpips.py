"""LPIPS on one GPU: this library's path (lpips_scores, bf16 and exact) against the torch chain a user would otherwise run
(torchvision's VGG16 features plus the LPIPS head in torch ops) on the same device and the same seeded weights, the chain in
three modes: fp32 with cuDNN's default TF32 (what the evaluation script's --precision full runs), fp32 with TF32 off, and
autocast fp16 (--precision autocast).  Prints one JSON object: ms per call (CUDA events over warmed loops of about half a
second), peak memory beyond the inputs, each mode's largest per-frame deviation from the fp64 oracle, the library's per-kernel
profile with the convolutions' achieved TFLOP/s against 989, and the card's name and power limit.

    python tools/bench_lpips.py [--out bench_lpips.json] [--no-oracle]

Every accuracy number comes from seeded weights (oracle/lpips_oracle.py): trained weights are not available offline."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.lpips_oracle import CONV_IDX, SLICE, lpips_fp64, script_inputs, synthetic_lpips_state  # noqa: E402
from vidtok_b200 import _native as N  # noqa: E402
from vidtok_b200.metrics import LPIPS, lpips_scores  # noqa: E402

WORKLOADS = [("8x3x17x256x256_fp32", (8, 3, 17, 256, 256), torch.float32),
             ("8x3x17x256x256_bf16_recon", (8, 3, 17, 256, 256), torch.bfloat16),
             ("1x3x17x1080x1920_fp32", (1, 3, 17, 1080, 1920), torch.float32)]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()
    except Exception:
        return torch.cuda.get_device_name()


def make_pair(shape, dtype):
    g = torch.Generator().manual_seed(0)
    B, Cc, T, H, W = shape
    coarse = torch.rand((B * Cc * T, 1, H // 16, W // 16), generator=g) * 2 - 1
    x = F.interpolate(coarse, size=(H, W), mode="bilinear", align_corners=False).reshape(shape) * 0.7
    x = (x + 0.1 * torch.randn(shape, generator=g)).clamp(-1, 1)
    y = 1.05 * x + 0.1 * torch.randn(shape, generator=g)
    return x.cuda(), y.to(dtype).cuda()


class TorchChain(torch.nn.Module):
    """torchvision's VGG16 features[0:30] and the LPIPS head in torch ops, per group of 16 frames as the script runs it"""

    def __init__(self, state):
        super().__init__()
        import torchvision
        net = torchvision.models.vgg16(weights=None).features[:30]
        net.load_state_dict({f"{i}.{p}": state[f"net.slice{s}.{i}.{p}"] for s, i in zip(SLICE, CONV_IDX) for p in ("weight", "bias")})
        self.net = net.eval().cuda()
        self.lin = [state[f"lin{k}.model.1.weight"].cuda() for k in range(5)]
        self.register_buffer("shift", torch.tensor([-.030, -.088, -.188]).view(1, 3, 1, 1).cuda())
        self.register_buffer("scale", torch.tensor([.458, .448, .450]).view(1, 3, 1, 1).cuda())
        self.taps = [3, 8, 15, 22, 29]

    def feats(self, v):
        out, h = [], v
        for i, layer in enumerate(self.net):
            h = layer(h)
            if i in self.taps:
                out.append(h)
        return out

    def forward(self, a, b):
        fa, fb = self.feats((a - self.shift) / self.scale), self.feats((b - self.shift) / self.scale)
        val = 0
        for k in range(5):
            na = fa[k] / (torch.sqrt((fa[k] ** 2).sum(1, keepdim=True)) + 1e-10)
            nb = fb[k] / (torch.sqrt((fb[k] ** 2).sum(1, keepdim=True)) + 1e-10)
            val = val + F.conv2d((na - nb) ** 2, self.lin[k].to(na.dtype)).mean((2, 3), keepdim=True)
        return val.flatten()


def chain_scores(chain, x, y, mode):
    frames = lambda t: t.permute(0, 2, 1, 3, 4).reshape(-1, t.shape[1], t.shape[3], t.shape[4])
    a, b = script_inputs(frames(x), frames(y))
    torch.backends.cudnn.allow_tf32 = mode == "fp32_tf32"
    out = []
    with torch.no_grad(), torch.autocast("cuda", enabled=mode == "autocast_fp16"):
        for i in range(0, a.shape[0], 16):
            out.append(chain(a[i:i + 16], b[i:i + 16]).float())
    torch.backends.cudnn.allow_tf32 = True
    return torch.cat(out)


def timed(fn, target_s=0.5):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    n = max(2, int(target_s * 1000 / max(e0.elapsed_time(e1), 1e-3)))
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def peak_beyond(fn, base):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def fp64_oracle(state64, x, y):
    frames = lambda t: t.permute(0, 2, 1, 3, 4).reshape(-1, t.shape[1], t.shape[3], t.shape[4])
    fx, fy = frames(x), frames(y)
    out = []
    with torch.no_grad():
        for i in range(fx.shape[0]):
            out.append(lpips_fp64(state64, fx[i:i + 1], fy[i:i + 1])[0].cpu())
    return torch.cat(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-oracle", action="store_true", help="skip the fp64 deviations")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lpips measures on the GPU; no CUDA device is visible")
    state = synthetic_lpips_state(0)
    state_dev = {k: v.cuda() for k, v in state.items()}
    models = {p: LPIPS.from_state_dict(state, precision=p) for p in ("bf16", "exact")}
    chain = TorchChain(state)
    result = {"card": card(), "weights": "synthetic_lpips_state(0) (seeded, not trained)", "workloads": {}}
    for name, shape, ydt in WORKLOADS:
        x, y = make_pair(shape, ydt)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        ref = None if args.no_oracle else fp64_oracle(state_dev, x, y)
        row = {}
        for p, m in models.items():
            fn = lambda m=m: lpips_scores(m, x, y)
            got = fn().reshape(-1).double().cpu()
            row[f"lib_{p}"] = {"ms": timed(fn), "peak_mib": peak_beyond(fn, base),
                               "max_abs_dev_fp64": None if ref is None else float((got - ref.double()).abs().max())}
            N.lib().vt_profile_start()
            fn()
            buf = C.create_string_buffer(1 << 20)
            N.lib().vt_profile_stop(buf, len(buf))
            prof = json.loads(buf.value.decode())
            conv = [v for k, v in prof.items() if k.startswith(("conv_tc", "lpips_stem"))]
            ms, fl = sum(v["ms"] for v in conv), sum(v["flops"] for v in conv)
            row[f"lib_{p}"]["profile"] = prof
            row[f"lib_{p}"]["conv_tflops"] = fl / ms / 1e9 if ms else None
            row[f"lib_{p}"]["conv_share_of_989"] = fl / ms / 1e9 / 989 if ms else None
        for mode in ("fp32_tf32", "fp32_no_tf32", "autocast_fp16"):
            fn = lambda mode=mode: chain_scores(chain, x, y, mode)
            got = fn().double().cpu()
            row[f"torch_{mode}"] = {"ms": timed(fn), "peak_mib": peak_beyond(fn, base),
                                    "max_abs_dev_fp64": None if ref is None else float((got - ref.double()).abs().max())}
        row["fp64_mean"] = None if ref is None else float(ref.mean())
        result["workloads"][name] = row
        print(name, json.dumps({k: (v["ms"], v["peak_mib"], v["max_abs_dev_fp64"]) for k, v in row.items() if isinstance(v, dict)}), flush=True)
        del x, y
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps({"card": result["card"]}))


if __name__ == "__main__":
    main()
