"""Time one conv geometry on the wgmma path (CUDA events, 20 launches).
usage: python tools/bench_conv.py Ci Co kt kh kw B T H W [res]"""
import ctypes as C
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vidtok_b200 import _native as N

Ci, Co, kt, kh, kw, B, T, H, W = [int(a) for a in sys.argv[1:10]]
res_mode = int(sys.argv[10]) if len(sys.argv) > 10 else 0
d = N.ConvDesc()
d.B, d.Ti, d.Hi, d.Wi, d.Ci, d.Co = B, T, H, W, Ci, Co
d.kt, d.kh, d.kw = kt, kh, kw
d.st = d.sh = d.sw = 1
d.pt = kt - 1
d.ph0 = d.ph1 = (kh - 1) // 2
d.pw0 = d.pw1 = (kw - 1) // 2
d.ut = d.uh = d.uw = 1
d.res_mode, d.alpha = res_mode, 0.0
x = torch.randn(B, T, H, W, Ci, device="cuda").bfloat16()
w = (torch.randn(Co, Ci, kt, kh, kw, device="cuda") / (Ci * kt * kh * kw) ** 0.5)
b = torch.randn(Co, device="cuda")
r = torch.randn(B, T, H, W, Co, device="cuda").bfloat16() if res_mode else None
out = torch.empty(B, T, H, W, Co, device="cuda", dtype=torch.bfloat16)
lib = N.lib()


def run():
    N.check(lib.vt_op_conv(N.PREC_BF16, 0, C.byref(d), C.c_void_p(x.data_ptr()), C.c_void_p(w.data_ptr()), C.c_void_p(b.data_ptr()),
                           C.c_void_p(r.data_ptr() if r is not None else 0), C.c_void_p(out.data_ptr()), None))


buf = C.create_string_buffer(1 << 16)
for _ in range(3):
    run()
lib.vt_profile_start_detailed()
for _ in range(10):
    run()
lib.vt_profile_stop(buf, len(buf))
import json
prof = json.loads(buf.value.decode())
for k, v in prof.items():
    if k.startswith("conv_tc"):
        print(f"{v['ms'] / v['launches']:.4f} ms  {v['flops'] / v['ms'] / 1e9:.1f} TF/s  {k}")
