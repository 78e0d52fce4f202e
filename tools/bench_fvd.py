"""I3D features for FVD on one GPU: this library's path (i3d_features, bf16 and exact) against the same network in torch ops on
the same device and the same seeded weights, in three modes: fp32 with cuDNN's default TF32, fp32 with TF32 off, and autocast
fp16.  Prints one JSON object per workload: ms per call (CUDA events over warmed loops of about half a second), peak memory
beyond the inputs, each mode's largest feature deviation from the fp64 oracle relative to the features' max |value|, the
library's per-kernel profile with the convolutions' achieved TFLOP/s, and the card's name and power limit.

    python tools/bench_fvd.py [--out bench_fvd.json] [--no-oracle]

Every accuracy number comes from seeded weights (oracle/i3d_oracle.py): trained weights are not available offline."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.i3d_oracle import _I3D_MODULES, _pool, _same_pad, i3d_fp64, preprocess, synthetic_i3d_state  # noqa: E402
from tools.bench_lpips import card, peak_beyond, timed  # noqa: E402
from vidtok_b200 import _native as N  # noqa: E402
from vidtok_b200.metrics import I3D, i3d_features  # noqa: E402

WORKLOADS = [("8x3x17x256x256", (8, 3, 17, 256, 256)), ("1x3x17x1080x1920", (1, 3, 17, 1080, 1920))]


def make_clips(shape):
    g = torch.Generator().manual_seed(0)
    B, Cc, T, H, W = shape
    coarse = torch.rand((B * Cc, T, H // 32, W // 32), generator=g) * 2 - 1
    x = F.interpolate(coarse, size=(H, W), mode="bilinear", align_corners=False).reshape(shape) * 0.8
    return (x + 0.05 * torch.randn(shape, generator=g)).clamp(-1, 1).cuda()


def torch_features(sd, x, mode):
    """the oracle's network in the given torch mode, BatchNorm folded as the library folds it"""
    torch.backends.cudnn.allow_tf32 = mode == "fp32_tf32"
    with torch.no_grad(), torch.autocast("cuda", enabled=mode == "autocast_fp16"):
        def unit(h, key, k, s=1):
            return F.relu(F.conv3d(_same_pad(h, (k,) * 3, (s,) * 3), sd[key][0], sd[key][1], stride=s))
        h = unit(preprocess(x), "Conv3d_1a_7x7", 7, 2)
        h = _pool(h, (1, 3, 3), (1, 2, 2))
        h = unit(unit(h, "Conv3d_2b_1x1", 1), "Conv3d_2c_3x3", 3)
        h = _pool(h, (1, 3, 3), (1, 2, 2))
        for name, _ in _I3D_MODULES:
            if name == "Mixed_4b":
                h = _pool(h, (3, 3, 3), (2, 2, 2))
            if name == "Mixed_5b":
                h = _pool(h, (2, 2, 2), (2, 2, 2))
            h = torch.cat([unit(h, f"{name}.b0", 1), unit(unit(h, f"{name}.b1a", 1), f"{name}.b1b", 3),
                           unit(unit(h, f"{name}.b2a", 1), f"{name}.b2b", 3), unit(_pool(h, (3, 3, 3), (1, 1, 1)), f"{name}.b3b", 1)], 1)
        h = F.conv3d(F.avg_pool3d(h, (2, 7, 7), stride=1), sd["logits"][0], sd["logits"][1])
        out = h.squeeze(4).squeeze(3).mean(2).float()
    torch.backends.cudnn.allow_tf32 = True
    return out


def folded(state):
    sd = {}
    for key in {k.rsplit(".", 2)[0] for k in state if k.endswith("conv3d.weight")}:
        w = state[f"{key}.conv3d.weight"].double()
        if key == "logits":
            sd[key] = (w.float().cuda(), state["logits.conv3d.bias"].cuda())
            continue
        sc = state[f"{key}.bn.weight"].double() / (state[f"{key}.bn.running_var"].double() + 1e-3).sqrt()
        b = state[f"{key}.bn.bias"].double() - state[f"{key}.bn.running_mean"].double() * sc
        sd[key] = ((w * sc.view(-1, 1, 1, 1, 1)).float().cuda(), b.float().cuda())
    return sd


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-oracle", action="store_true", help="skip the fp64 deviations")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fvd measures on the GPU; no CUDA device is visible")
    state = synthetic_i3d_state(0)
    models = {p: I3D.from_state_dict(state, precision=p) for p in ("bf16", "exact")}
    sd = folded(state)
    result = {"card": card(), "weights": "synthetic_i3d_state(0) (seeded, not trained)", "workloads": {}}
    for name, shape in WORKLOADS:
        x = make_clips(shape)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        ref = None
        if not args.no_oracle:
            with torch.no_grad():
                ref = torch.cat([i3d_fp64(state, x[i:i + 1])[1].cpu() for i in range(shape[0])])
        dev = lambda got: None if ref is None else float((got.double().cpu() - ref).abs().max() / ref.abs().max())
        row = {}
        for p, m in models.items():
            fn = lambda m=m: i3d_features(m, x)
            got = fn()
            row[f"lib_{p}"] = {"ms": timed(fn), "peak_mib": peak_beyond(fn, base), "rel_dev_fp64": dev(got)}
            N.lib().vt_profile_start()
            fn()
            buf = C.create_string_buffer(1 << 20)
            N.lib().vt_profile_stop(buf, len(buf))
            prof = json.loads(buf.value.decode())
            conv = [v for k, v in prof.items() if k.startswith(("conv_tc", "i3d_stem"))]
            ms, fl = sum(v["ms"] for v in conv), sum(v["flops"] for v in conv)
            row[f"lib_{p}"]["profile"] = prof
            row[f"lib_{p}"]["conv_tflops"] = fl / ms / 1e9 if ms else None
        for mode in ("fp32_tf32", "fp32_no_tf32", "autocast_fp16"):
            fn = lambda mode=mode: torch_features(sd, x, mode)
            got = fn()
            row[f"torch_{mode}"] = {"ms": timed(fn), "peak_mib": peak_beyond(fn, base), "rel_dev_fp64": dev(got)}
        result["workloads"][name] = row
        print(name, json.dumps({k: (round(v["ms"], 2), round(v["peak_mib"]), v["rel_dev_fp64"]) for k, v in row.items()}), flush=True)
        del x
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps({"card": result["card"]}))


if __name__ == "__main__":
    main()
