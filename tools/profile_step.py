"""Per-layer timing of one forward (detailed profiler keys) -- run on a GPU machine.
  python tools/profile_step.py [B] [bf16|exact|mixed|fma] [kl488|fsq488|v11long|kl41616]"""
import ctypes
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from vidtok_b200 import _native as N  # noqa: E402
if os.environ.get("VT_AB_LIB"):   # same-run A/B against another build of the library (development only)
    N.LIB_PATH = os.environ["VT_AB_LIB"]
from vidtok_b200.compat_util import instantiate_from_config  # noqa: E402
from vidtok_b200.synth import synth_clip, synth_state_dict  # noqa: E402


def main():
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 8
    prec = sys.argv[2] if len(sys.argv) > 2 else "bf16"
    cfg_name = sys.argv[3] if len(sys.argv) > 3 else "kl488"
    c = bench.CONFIGS[cfg_name]
    model = instantiate_from_config(bench.model_cfg(c))
    sd = synth_state_dict({k: tuple(v.shape) for k, v in model.state_dict().items()}, seed=0)
    model.load_state_dict(sd)
    model = model.cuda().eval()
    model.precision = prec
    if c["tiling"]:
        model.use_tiling = True
        model.t_chunk_enc, model.t_chunk_dec, model.use_overlap = c["tiling"]
    x = synth_clip(B, c["T"], c["H"], c["W"]).cuda()
    with torch.no_grad():
        for _ in range(2):
            model(x)
        torch.cuda.synchronize()
        lib = N.lib()
        lib.vt_profile_start_detailed()
        model(x)
        buf = ctypes.create_string_buffer(1 << 20)
        n = lib.vt_profile_stop(buf, len(buf))
    prof = json.loads(buf.value.decode())
    tot = sum(v["ms"] for v in prof.values())
    print(f"total kernel ms {tot:.2f} over {sum(v['launches'] for v in prof.values())} launches")
    for k, v in sorted(prof.items(), key=lambda kv: -kv[1]["ms"])[:45]:
        tf = v["flops"] / (v["ms"] / 1e3) / 1e12 if v["flops"] else 0.0
        gb = v["bytes"] / (v["ms"] / 1e3) / 1e9 if v["bytes"] else 0.0
        print(f"{v['ms']:9.3f} ms  n={v['launches']:3d}  {tf:7.1f} TF/s {gb:8.0f} GB/s  {k}")


if __name__ == "__main__":
    main()
