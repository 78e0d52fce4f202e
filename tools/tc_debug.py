"""GPU-side diagnostics for the wgmma conv kernel: structured inputs that expose layout/descriptor mistakes
(row permutations, K-chunk swaps, swizzle mismatches) instead of a bare pass/fail.  Run on a GPU machine."""
import math
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from gpu_util import op_conv  # noqa: E402
from vidtok_b200 import _native as N  # noqa: E402


def ref_conv(x, w, b, stride=(1, 1, 1)):
    kt, kh, kw = w.shape[2:]
    tp = (kt - 1) + (1 - stride[0])
    x = F.pad(x, (kw // 2, kw // 2, kh // 2, kh // 2, tp, 0))
    return F.conv3d(x, w, b, stride=stride)


def report(name, got, ref):
    err = (got - ref).abs()
    print(f"[{name}] shape {tuple(got.shape)} max|err|={float(err.max()):.4e} mean|err|={float(err.mean()):.4e} "
          f"ref absmax={float(ref.abs().max()):.3f} got absmax={float(got.abs().max()):.3f} nan={int(torch.isnan(got).sum())}")
    return float(err.max())


def main():
    torch.manual_seed(0)
    g = torch.Generator().manual_seed(0)
    # 1) identity GEMM: 128 positions, 64 -> 64 channels, w = I : out must equal x (bf16-rounded)
    x = torch.randn(1, 64, 1, 8, 16, generator=g).bfloat16().float()
    w = torch.eye(64).reshape(64, 64, 1, 1, 1)
    got = op_conv(x, w, torch.zeros(64), precision=N.PREC_BF16)
    e = report("identity 1x1x1", got, x)
    if e > 1e-2:
        # which (position, channel) of the input does each output element equal?
        xf = x[0, :, 0].reshape(64, 128).t()  # [pos, ch]
        gf = got[0, :, 0].reshape(64, 128).t()
        for pos in (0, 1, 8, 17):
            for ch in (0, 1, 8, 33):
                m = (xf - gf[pos, ch]).abs() < 1e-6
                hits = m.nonzero().tolist()[:3]
                print(f"   out[pos={pos},ch={ch}]={float(gf[pos, ch]):+.4f} matches x at {hits}")
    # 2) random GEMM
    w = (torch.randn(64, 64, 1, 1, 1, generator=g) / 8).bfloat16().float()
    b = torch.randn(64, generator=g)
    report("random 1x1x1", op_conv(x, w, b, precision=N.PREC_BF16), ref_conv(x, w, b))
    # 3) one tap at a time of a 3x3 spatial conv (exposes coordinate / padding mistakes)
    x = torch.randn(1, 64, 2, 16, 16, generator=g).bfloat16().float()
    for tap in range(9):
        w = torch.zeros(64, 64, 1, 3, 3)
        w[:, :, 0, tap // 3, tap % 3] = torch.eye(64)
        report(f"3x3 tap {tap}", op_conv(x, w, torch.zeros(64), precision=N.PREC_BF16), ref_conv(x, w, torch.zeros(64)))
    # 4) temporal taps
    for tap in range(3):
        w = torch.zeros(64, 64, 3, 1, 1)
        w[:, :, tap, 0, 0] = torch.eye(64)
        report(f"3x1x1 tap {tap}", op_conv(x, w, torch.zeros(64), precision=N.PREC_BF16), ref_conv(x, w, torch.zeros(64)))
    # 5) K = 2 chunks, N = 128
    x = torch.randn(1, 128, 1, 16, 16, generator=g).bfloat16().float()
    w = (torch.randn(128, 128, 1, 3, 3, generator=g) / math.sqrt(128 * 9)).bfloat16().float()
    b = torch.randn(128, generator=g)
    report("3x3 C128", op_conv(x, w, b, precision=N.PREC_BF16), ref_conv(x, w, b))
    # 6) many tiles, persistent loop with phase wrap
    x = torch.randn(2, 64, 4, 64, 64, generator=g).bfloat16().float()
    w = (torch.randn(64, 64, 3, 3, 3, generator=g) / math.sqrt(64 * 27)).bfloat16().float()
    b = torch.randn(64, generator=g)
    report("3x3x3 many tiles", op_conv(x, w, b, precision=N.PREC_BF16), ref_conv(x, w, b))
    print("tc_debug done")


if __name__ == "__main__":
    main()
