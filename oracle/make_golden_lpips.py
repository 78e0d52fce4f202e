"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/lpips/*.npz: per-frame LPIPS of the UNMODIFIED reference
vidtok.modules.lpips.LPIPS (imported through oracle/ref_shim.py) with the seeded weights of oracle/lpips_oracle.py, in fp32 and
in fp64, next to the fp64 oracle's five layer terms.

Needs the reference checkout and torchvision:   python oracle/make_golden_lpips.py

Nothing here reaches the network.  In the loaded reference module only `models` (torchvision.models) is replaced, by a namespace
whose vgg16() returns torchvision's VGG16 with the seeded features; the seeded lin weights are written to
checkpoints/lpips/vgg.pth in a temporary working directory, where get_ckpt_path finds an existing file.

Each file holds frame pairs x, y [N,3,H,W] (fp32, y not yet clamped) of one size covering: x == y, a small and a large
distortion, a reconstruction with values outside [-1,1], and a bf16 reconstruction (y exactly representable in bf16; the GPU
test passes that frame as a bfloat16 tensor).
"""
from __future__ import annotations

import json
import os
import sys
import tempfile
import types
import warnings

warnings.filterwarnings("ignore")

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402
from oracle.lpips_oracle import CONV_IDX, SLICE, lpips_fp64, script_inputs, synthetic_lpips_state  # noqa: E402

OUT = os.environ.get("VIDTOK_GOLDEN_LPIPS_OUT", os.path.join(ROOT, "tests", "golden", "lpips"))
WEIGHT_SEED = 0
CASES = ("equal", "small", "large", "out_of_range", "bf16")
SIZES = ((64, 64, 11), (48, 80, 12))   # H, W, input seed


def make_inputs(H, W, seed):
    g = torch.Generator().manual_seed(seed)
    # a smooth image plus texture, in [-1, 1]
    base = torch.nn.functional.interpolate(torch.rand(1, 3, H // 8, W // 8, generator=g) * 2 - 1, size=(H, W), mode="bilinear",
                                           align_corners=False)
    x = (0.7 * base + 0.3 * (torch.rand(1, 3, H, W, generator=g) * 2 - 1)).clamp(-1, 1).repeat(len(CASES), 1, 1, 1)
    y = x.clone()
    y[1] = x[1] + 0.01 * torch.randn(3, H, W, generator=g)
    y[2] = x[2] + 0.3 * torch.randn(3, H, W, generator=g)
    y[3] = 1.4 * x[3] + 0.05 * torch.randn(3, H, W, generator=g)
    y[4] = (x[4] + 0.1 * torch.randn(3, H, W, generator=g)).to(torch.bfloat16).float()
    return x.contiguous(), y.contiguous()


def reference_model(state):
    import torchvision

    ref_shim.import_reference()
    import vidtok.modules.lpips as L

    def vgg16(pretrained=True, **kw):
        net = torchvision.models.vgg16(weights=None)
        feats = {f"features.{i}.{p}": state[f"net.slice{s}.{i}.{p}"] for s, i in zip(SLICE, CONV_IDX) for p in ("weight", "bias")}
        net.load_state_dict(feats, strict=False)
        return net

    L.models = types.SimpleNamespace(vgg16=vgg16)
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "checkpoints", "lpips"))
        torch.save({k: v for k, v in state.items() if k.startswith("lin")}, os.path.join(tmp, "checkpoints", "lpips", "vgg.pth"))
        os.chdir(tmp)
        try:
            model = L.LPIPS().eval()
        finally:
            os.chdir(cwd)
    for k, v in model.state_dict().items():
        if k in state:
            assert torch.equal(v, state[k]), k
    return model


def main():
    state = synthetic_lpips_state(WEIGHT_SEED)
    model = reference_model(state)
    os.makedirs(OUT, exist_ok=True)
    for H, W, seed in SIZES:
        x, y = make_inputs(H, W, seed)
        a, b = script_inputs(x, y)
        with torch.no_grad():
            ref32 = model(a, b).flatten()
            ref64 = model.double()(a.double(), b.double()).flatten()
            model.float()
        total, per_layer = lpips_fp64(state, x, y)
        dev = float((total - ref64).abs().max())
        assert dev <= 1e-12, f"oracle against the reference's fp64 forward: {dev:.3e}"
        meta = {"weight_seed": WEIGHT_SEED, "input_seed": seed, "cases": list(CASES), "oracle_vs_reference_fp64": dev,
                "fp32_vs_fp64": float((ref32.double() - ref64).abs().max())}
        name = f"lpips_{H}x{W}"
        np.savez_compressed(os.path.join(OUT, name + ".npz"), x=x.numpy(), y=y.numpy(), ref_fp32=ref32.numpy(),
                            ref_fp64=ref64.numpy(), layers_fp64=per_layer.numpy(),
                            meta_json=np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8))
        print(f"[lpips] {name}: fp64 {np.array2string(ref64.numpy(), precision=6)} oracle dev {dev:.2e} "
              f"fp32 dev {meta['fp32_vs_fp64']:.2e}", flush=True)


if __name__ == "__main__":
    main()
