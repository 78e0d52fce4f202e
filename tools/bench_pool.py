"""Many feeds of different lengths with staggered starts, encoded and decoded three ways on one GPU:

  pool    one EncodePool + one DecodePool (vidtok_b200.streaming) holding every feed in flight;
  streams one EncodeStream + DecodeStream of batch 1 per feed, driven in the same interleaved order;
  tile    tile_encode + tile_decode per video, one video after another.

kl_causal_488_4chn_v1_1 with synthetic weights (seed 0), the long-video recipe (t_chunk_enc 16, t_chunk_dec 4,
use_overlap), bf16 by default.  Feed i has a length drawn from [--min-frames, --max-frames] (seed 0), opens at step
i * --stagger and pushes --push frames per step until it ends; its latents go to the decoder in the step they appear.
Each way runs in a process of its own (so its memory starts from the same baseline), once untimed and once timed with CUDA
events around the whole workload.  Reported per way: frames/s (all feeds' frames over the timed run), the peak of the
torch allocator above the start (workspaces, staged chunks, outputs), the peak device memory in use above the start
(cudaMemGetInfo after every step: adds the library's chunk caches), and for the pool the fraction of batched slot-chunks
that carried no video (idle or zero-fed slots) and the time in slot transplants (CUDA events around each
vt_chunk_state_copy_slots).  The card's name, power limit and SM clocks are read in the same process.

    python tools/bench_pool.py [--feeds 16] [--size 128] [--min-frames 33] [--max-frames 257] [--precision bf16]
"""
import argparse
import gzip
import json
import os
import random
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, power, sm, sm_max = [v.strip() for v in q.split(",")]
    return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


def feeds(a):
    rng = random.Random(0)
    return [(i * a.stagger, rng.randint(a.min_frames, a.max_frames)) for i in range(a.feeds)]


def run_way(a):
    import torch
    from vidtok_b200.compat_util import instantiate_from_config
    from vidtok_b200.streaming import DecodePool, DecodeStream, EncodePool, EncodeStream
    from vidtok_b200.synth import synth_state_dict
    if not torch.cuda.is_available():
        raise SystemExit("bench_pool needs a CUDA device")
    zoo = json.load(gzip.open(os.path.join(ROOT, "tests", "golden", "zoo_manifest.json.gz"), "rt"))
    rec = zoo["vidtok_v1_1/vidtok_kl_causal_488_4chn_v1_1.yaml"]
    model = instantiate_from_config(rec["model"])
    model.load_state_dict(synth_state_dict({k: tuple(v) for k, v in rec["shapes"].items()}, seed=0), strict=False)
    model = model.to("cuda").eval()
    model.precision = a.precision
    model.use_tiling, model.t_chunk_enc, model.t_chunk_dec, model.use_overlap = True, 16, 4, True
    plan = feeds(a)
    g = torch.Generator().manual_seed(1)
    xs = [(torch.rand((1, 3, T, a.size, a.size), generator=g) * 2 - 1).cuda() for _, T in plan]
    total = sum(T for _, T in plan)
    nat = model._rt.sync()
    Hz = nat.latent_shape(1, a.size, a.size)[1]
    capacity = max(sum(1 for s, T in plan if s <= t < s + -(-T // a.push)) for t in range(plan[-1][0] + 1))
    free0 = torch.cuda.mem_get_info()[0]
    peak_dev = [0]

    def sample():
        peak_dev[0] = max(peak_dev[0], free0 - torch.cuda.mem_get_info()[0])

    tx = {"events": []}

    def workload():
        if a.way == "tile":
            for x in xs:
                z, _ = model.tile_encode(x)
                model.tile_decode(z)
                sample()
            return None
        if a.way == "pool":
            enc = EncodePool(model, capacity, a.size, a.size, t_chunk=16)
            dec = DecodePool(model, capacity, Hz, Hz, t_chunk=4, use_overlap=True)
            for p in (enc, dec):
                copy = p._copy

                def timed_copy(*args, _copy=copy):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    _copy(*args)
                    e1.record()
                    tx["events"].append((e0, e1))
                p._copy = timed_copy
        open_, t0, step = {}, {}, 0
        while len(t0) < len(plan) or open_:
            for i, (start, T) in enumerate(plan):
                if start == step:
                    if a.way == "pool":
                        open_[i] = (enc.open(), dec.open())
                    else:
                        open_[i] = (EncodeStream(model, 1, a.size, a.size, t_chunk=16),
                                    DecodeStream(model, 1, Hz, Hz, t_chunk=4, use_overlap=True))
                    t0[i] = 0
            done = []
            for i, (e, d) in open_.items():
                T = plan[i][1]
                n = min(a.push, T - t0[i])
                if a.way == "pool":
                    enc.push(e, xs[i][:, :, t0[i]:t0[i] + n])
                else:
                    z, _ = e.push(xs[i][:, :, t0[i]:t0[i] + n])
                    d.push(z)
                t0[i] += n
                if t0[i] == T:
                    done.append(i)
            if a.way == "pool":
                slot_feed = {e: i for i, (e, _) in open_.items()}
                for s, (z, _) in enc.step().items():
                    dec.push(open_[slot_feed[s]][1], z)
                dec.step()
            for i in done:
                e, d = open_.pop(i)
                if a.way == "pool":
                    z, _ = enc.close(e)
                    if z.shape[2]:
                        dec.push(d, z)
                    dec.close(d)
                else:
                    z, _ = e.flush()
                    d.push(z)
                    d.flush()
                    e.close()
                    d.close()
            sample()
            step += 1
        if a.way == "pool":
            stats = {"enc": dict(enc.counts), "dec": dict(dec.counts), "capacity": capacity}
            enc.close_pool()
            dec.close_pool()
            return stats
        return None

    with torch.no_grad():
        workload()
        torch.cuda.synchronize()
        tx["events"].clear()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        stats = workload()
        e1.record()
        torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    out = {"way": a.way, "model": "kl_causal_488_4chn_v1_1 (synthetic weights)", "precision": a.precision,
           "size": a.size, "feeds": a.feeds, "frames": total, "lengths": [T for _, T in plan], "stagger_steps": a.stagger,
           "push": a.push, "ms": round(ms, 1), "frames_per_s": round(total / (ms / 1e3), 1),
           "peak_torch_gb": round((torch.cuda.max_memory_allocated() - base) / 2**30, 3),
           "peak_device_gb": round(peak_dev[0] / 2**30, 3), "card": card()}
    if stats:
        for k in ("enc", "dec"):
            c = stats[k]
            slots = c["batched"] * stats["capacity"]
            out[k] = {**c, "idle_fraction": round(1 - c["slot_chunks"] / slots, 3) if slots else None}
        out["capacity"] = stats["capacity"]
        out["transplant_ms"] = round(sum(s.elapsed_time(e) for s, e in tx["events"]), 2)
        out["transplant_share"] = round(out["transplant_ms"] / ms, 4)
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--feeds", type=int, default=16)
    ap.add_argument("--size", type=int, default=128)
    ap.add_argument("--min-frames", type=int, default=33)
    ap.add_argument("--max-frames", type=int, default=257)
    ap.add_argument("--stagger", type=int, default=1, help="steps between two feeds' starts")
    ap.add_argument("--push", type=int, default=16, help="frames each feed pushes per step")
    ap.add_argument("--precision", default="bf16")
    ap.add_argument("--ways", default="pool,streams,tile")
    ap.add_argument("--way", default=None, help=argparse.SUPPRESS)   # one way, in this process
    a = ap.parse_args()
    if a.way:
        run_way(a)
        return
    for way in a.ways.split(","):
        args = [sys.executable, os.path.abspath(__file__), "--way", way] + sys.argv[1:]
        subprocess.run(args, check=True)


if __name__ == "__main__":
    main()
