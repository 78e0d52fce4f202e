"""Streamed vs whole-clip encode of kl_causal_488_4chn (synthetic weights): per-push latency (CUDA events), frames/s and the
peak workspace of each configuration (vt_chunk_workspace_bytes / vt_workspace_bytes dry runs), for

  256x256 B=8 bf16    pushes of 4 frames and of 16 frames (after the 1-frame first push), and the whole clip
  720x1280 B=1 bf16   pushes of 4 frames, and the whole clip
  1080x1920 B=1 exact pushes of 4 frames only (the whole clip needs more workspace than an 80 GB card has)
  1080x1920 B=1 bf16  pushes of 4 frames only

Frames/s counts input frames of the steady pushes (the first 1-frame push is timed apart).  Prints one JSON line per
configuration and the card, its power limit and SM clocks.
usage: python tools/bench_stream.py [--clips 2] [--lib PATH] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vidtok_b200 import _native as N  # noqa: E402
from vidtok_b200.streaming import EncodeStream  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[torch.cuda.current_device()]
    except Exception as e:
        return f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {e})"


def kl488():
    from oracle.make_golden import model_yaml
    from vidtok_b200.compat_util import instantiate_from_config
    from vidtok_b200.synth import synth_state_dict
    cfg = model_yaml(version="v1_0", reg="kl", ch=128, ch_mult=(1, 2, 4, 4), z=4, interp=None)
    cfg["params"]["decoder_config"]["params"] = dict(cfg["params"]["encoder_config"]["params"])
    cfg["params"]["regularizer_config"]["params"] = {"sample": False}
    model = instantiate_from_config(cfg)
    model.load_state_dict(synth_state_dict({k: tuple(v.shape) for k, v in model.state_dict().items()}, seed=0))
    return model.cuda().eval()


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def stream_run(model, B, H, W, push, pushes, clips):
    """clips x (1 + pushes * push frames); returns first-push ms, steady per-push ms list, peak workspace bytes"""
    x = torch.randn((B, 3, push, H, W), device="cuda").clamp_(-1, 1)
    x1 = x[:, :, :1].contiguous()
    enc = EncodeStream(model, B, H, W)
    lib = N.lib()
    ws = max(lib.vt_chunk_workspace_bytes(enc.state.handle, 1), lib.vt_chunk_workspace_bytes(enc.state.handle, push))
    first, steady = [], []
    for c in range(clips + 1):          # clip 0 warms up every shape
        enc.reset()
        f = timed(lambda: enc.push(x1))
        s = [timed(lambda: enc.push(x)) for _ in range(pushes)]
        if c:
            first.append(f)
            steady += s
    enc.close()
    return sum(first) / len(first), steady, ws


def whole_run(model, B, H, W, T, clips):
    x = torch.randn((B, 3, T, H, W), device="cuda").clamp_(-1, 1)
    ws = N.lib().vt_workspace_bytes(model._rt.sync().handle, model._rt.precision(), B, T, H, W)
    ms = [timed(lambda: model.encode(x)) for _ in range(clips + 1)][1:]
    return sum(ms) / len(ms), ws


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=2)
    ap.add_argument("--out", default=None)
    ap.add_argument("--lib", default=None, help="library to measure (default: the in-tree build)")
    args = ap.parse_args()
    if args.lib:
        N.LIB_PATH = os.path.abspath(args.lib)
    if not torch.cuda.is_available():
        raise SystemExit("bench_stream: no CUDA device; these numbers need an H100")
    model = kl488()
    rows = []
    with torch.no_grad():
        for (B, H, W, prec, pushes, whole) in ((8, 256, 256, "bf16", (4, 16), True), (1, 720, 1280, "bf16", (4,), True),
                                               (1, 1080, 1920, "exact", (4,), False), (1, 1080, 1920, "bf16", (4,), False)):
            model.precision = prec
            T = 17
            if whole:
                ms, ws = whole_run(model, B, H, W, T, args.clips)
                rows.append({"config": f"{H}x{W} B={B} {prec}", "run": f"whole clip T={T}", "ms_per_clip": round(ms, 2),
                             "frames_per_s": round(B * T / ms * 1e3, 1), "workspace_GB": round(ws / 1e9, 2)})
                model._rt.native._ws = None
                torch.cuda.empty_cache()
            for push in pushes:
                n = (T - 1) // push
                first, steady, ws = stream_run(model, B, H, W, push, n, args.clips)
                ms = sum(steady) / len(steady)
                rows.append({"config": f"{H}x{W} B={B} {prec}", "run": f"stream 1 + {n}x{push}", "first_push_ms": round(first, 2),
                             "ms_per_push": round(ms, 2), "max_push_ms": round(max(steady), 2),
                             "frames_per_s": round(B * push / ms * 1e3, 1), "workspace_GB": round(ws / 1e9, 2)})
                model._rt.native._ws = None
                torch.cuda.empty_cache()
    out = {"card": card(), "model": "kl_causal_488_4chn (synthetic weights)", "rows": rows}
    for r in rows:
        print(json.dumps(r))
    print(json.dumps({"card": out["card"]}))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
