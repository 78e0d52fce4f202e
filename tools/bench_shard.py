"""One long video as shards in one batch (vidtok_b200.longvideo) against tile_encode + tile_decode on one GPU.

kl_causal_488_4chn_v1_1 with synthetic weights (seed 0), t_chunk_enc 16, t_chunk_dec 4, use_overlap, bf16 by default.  For
each shard count: encode + decode frames/s of the whole video (CUDA events, after one untimed run of the same call), the
plan's warm-up fraction in each direction, and the peak device memory of the call.  The card's name, power limit and SM
clock are read in the same run.  Prints one JSON line per configuration.

    python tools/bench_shard.py [--frames 1025] [--size 256] [--shards 1,2,4,8] [--precision bf16]
"""
import argparse
import gzip
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, power, sm, sm_max = [v.strip() for v in q.split(",")]
    return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


def main():
    import torch
    from vidtok_b200.compat_util import instantiate_from_config
    from vidtok_b200.longvideo import decode_sharded, encode_sharded, shard_plan, temporal_reach
    from vidtok_b200.synth import synth_state_dict
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1025)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--shards", default="1,2,4,8")
    ap.add_argument("--precision", default="bf16")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_shard needs a CUDA device")
    zoo = json.load(gzip.open(os.path.join(ROOT, "tests", "golden", "zoo_manifest.json.gz"), "rt"))
    rec = zoo["vidtok_v1_1/vidtok_kl_causal_488_4chn_v1_1.yaml"]
    model = instantiate_from_config(rec["model"])
    model.load_state_dict(synth_state_dict({k: tuple(v) for k, v in rec["shapes"].items()}, seed=0), strict=False)
    model = model.to("cuda").eval()
    model.precision, model.use_overlap = a.precision, True
    g = torch.Generator().manual_seed(0)
    x = (torch.rand((1, 3, a.frames, a.size, a.size), generator=g) * 2 - 1).cuda()
    nat = model._rt.sync()
    R_enc, R_dec = temporal_reach(nat, False), temporal_reach(nat, True, True)

    def timed(fn):
        fn()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), (torch.cuda.max_memory_allocated() - base) / 2**30

    def tile():
        torch.manual_seed(1)
        z, _ = model.tile_encode(x)
        model.tile_decode(z)

    ms, gb = timed(tile)
    base_fps = a.frames / (ms / 1e3)
    info = {"model": "kl_causal_488_4chn_v1_1 (synthetic weights)", "video": [1, 3, a.frames, a.size, a.size],
            "precision": a.precision, "reach": {"encoder_frames": R_enc, "decoder_latents_overlap": R_dec}, "card": card()}
    print(json.dumps({**info, "call": "tile_encode + tile_decode", "ms": round(ms, 1), "frames_per_s": round(base_fps, 1),
                      "peak_gb": round(gb, 2)}), flush=True)
    Tz = nat.latent_shape(a.frames, a.size, a.size)[0]
    for S in [int(s) for s in a.shards.split(",")]:
        try:
            pe = shard_plan(a.frames, S, model.t_chunk_enc, R_enc)
            pd = shard_plan(Tz, S, model.t_chunk_dec, R_dec, lookahead=True)
        except ValueError as e:
            print(json.dumps({**info, "shards": S, "refused": str(e)}), flush=True)
            continue

        def sharded():
            torch.manual_seed(1)
            z, _ = encode_sharded(model, x, S)
            decode_sharded(model, z, S)

        ms, gb = timed(sharded)
        print(json.dumps({**info, "call": "encode_sharded + decode_sharded", "shards": S, "ms": round(ms, 1),
                          "frames_per_s": round(a.frames / (ms / 1e3), 1), "vs_tile": round(a.frames / (ms / 1e3) / base_fps, 3),
                          "warmup_fraction": {"encoder": round(pe.warmup_fraction, 3), "decoder": round(pd.warmup_fraction, 3)},
                          "window": {"encoder_frames": pe.window, "decoder_latents": pd.window}, "peak_gb": round(gb, 2),
                          "card_after": card()}), flush=True)


if __name__ == "__main__":
    main()
