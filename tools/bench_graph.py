"""Host cost of a stream push, and what replaying CUDA graphs saves.

kl_causal_488_4chn_v1_1 with synthetic weights (seed 0), bf16, batch 1.  Workloads:
  enc4 / enc16   EncodeStream (no t_chunk: each push is one chunk) with pushes of 4 and of 16 frames;
  dec1           DecodeStream(t_chunk=4, use_overlap=True) with pushes of 1 latent frame (a chunk every 4th push);
at --sizes (default 128x128, 256x256, 720x1280; dec1 up to 256x256), and a whole-clip model(x) of 1x17x256x256 captured in a torch.cuda.graph
against the eager call.

Each stream workload runs two streams in one process: "eager" with graph replay switched off, "replay" as shipped (its
steady chunks replay captured graphs).  After a warm-up that captures every graph, the two alternate for --rounds rounds
of at least --seconds each.  Per push: host wall time of the push ended by a device synchronise; device time from CUDA
events around the push; enqueue time (the host time of the push call alone, without the synchronise); library kernel
launches per chunk (vt_launch_count: a replayed chunk launches one graph and no kernel of its own).  The card's name,
power limit and SM clocks are read in the same process.

    python tools/bench_graph.py [--sizes 128x128,256x256,720x1280] [--seconds 0.5] [--rounds 2] [--json out.json]
"""
import argparse
import gzip
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, power, sm, sm_max = [v.strip() for v in q.split(",")]
    return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


def load_model():
    import torch
    from vidtok_b200.compat_util import instantiate_from_config
    from vidtok_b200.synth import synth_state_dict
    zoo = json.load(gzip.open(os.path.join(ROOT, "tests", "golden", "zoo_manifest.json.gz"), "rt"))
    rec = zoo["vidtok_v1_1/vidtok_kl_causal_488_4chn_v1_1.yaml"]
    model = instantiate_from_config(rec["model"])
    model.load_state_dict(synth_state_dict({k: tuple(v) for k, v in rec["shapes"].items()}, seed=0), strict=False)
    model = model.to("cuda").eval()
    model.precision = "bf16"
    return model


def timed(push, seconds):
    """push() (which returns the chunks it ran) repeatedly for at least `seconds`: per push wall (synchronised), device
    (events) and enqueue times, and library launches per chunk"""
    import torch
    from vidtok_b200 import _native as N
    lib = N.lib()
    wall = dev = enq = 0.0
    pushes = chunks = launches = 0
    t_end = time.perf_counter() + seconds
    torch.cuda.synchronize()
    while time.perf_counter() < t_end or pushes < 8:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        lib.vt_launch_count(1)
        h0 = time.perf_counter()
        e0.record()
        n = push()
        e1.record()
        h1 = time.perf_counter()
        torch.cuda.synchronize()
        h2 = time.perf_counter()
        launches += lib.vt_launch_count(0)
        enq += h1 - h0
        wall += h2 - h0
        dev += e0.elapsed_time(e1) / 1e3
        pushes += 1
        chunks += n
    return {"pushes": pushes, "wall_ms": 1e3 * wall / pushes, "device_ms": 1e3 * dev / pushes, "enqueue_ms": 1e3 * enq / pushes,
            "launches_per_chunk": launches / max(chunks, 1), "chunks_per_push": chunks / pushes}


def stream_workload(model, kind, H, W, replay):
    import torch
    from vidtok_b200.streaming import DecodeStream, EncodeStream
    g = torch.Generator().manual_seed(1)
    if kind == "dec1":
        Hz, Wz = model._rt.sync().latent_shape(1, H, W)[1:]
        s = DecodeStream(model, 1, Hz, Wz, t_chunk=4, use_overlap=True)
        zs = [torch.randn((1, 4, 1, Hz, Wz), generator=g).cuda() for _ in range(8)]
        it = [0]

        def push():
            it[0] += 1
            return int(s.push(zs[it[0] % len(zs)]).shape[2] > 0)
    else:
        n = 4 if kind == "enc4" else 16
        s = EncodeStream(model, 1, H, W)
        xs = [(torch.rand((1, 3, n, H, W), generator=g) * 2 - 1).cuda() for _ in range(2)]
        s.push(xs[0][:, :, :1])   # the first chunk: frame 0 alone
        it = [0]

        def push():
            it[0] += 1
            s.push(xs[it[0] % 2])
            return 1
    if not replay:
        s.graphs.action = lambda key: "eager"
    return s, push


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="128x128,256x256,720x1280")
    ap.add_argument("--seconds", type=float, default=0.5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_graph needs a CUDA device")
    model = load_model()
    out = {"card": card(), "rows": []}
    print(json.dumps(out["card"]), flush=True)
    with torch.no_grad():
        for size in a.sizes.split(","):
            H, W = (int(v) for v in size.split("x"))
            for kind in ("enc4", "enc16", "dec1"):
                if kind == "dec1" and H * W > 256 * 256:
                    continue   # an eager and a replaying 720x1280 decode stream side by side do not fit in 80 GB
                model._rt.sync()._ws = None   # each workload sizes its own workspace (720x1280 ones are GBs)
                torch.cuda.empty_cache()
                ways = {}
                for replay in (False, True):
                    s, push = stream_workload(model, kind, H, W, replay)
                    for _ in range(24):   # warm-up: every graph key is captured (two cache parities)
                        push()
                    ways["replay" if replay else "eager"] = (s, push, [])
                for _ in range(a.rounds):
                    for name, (s, push, res) in ways.items():
                        res.append(timed(push, a.seconds))
                for name, (s, push, res) in ways.items():
                    row = {"workload": kind, "size": size, "way": name}
                    for k in res[0]:
                        row[k] = sum(r[k] for r in res) / len(res)
                    row["graphs"] = len(s.graphs.graphs)
                    out["rows"].append(row)
                    print(json.dumps(row), flush=True)
                    s.close()
        # whole clip: model(x) of 1x17x256x256 (untiled) captured in the caller's graph against eager
        model.use_tiling = False
        x = (torch.rand((1, 3, 17, 256, 256), generator=torch.Generator().manual_seed(2)) * 2 - 1).cuda()
        noise = torch.randn((1, 4, 5, 32, 32), generator=torch.Generator().manual_seed(3)).cuda()
        model(x, noise=noise)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            model(x, noise=noise)
        ways = {"eager": (lambda: model(x, noise=noise) and 1, []), "replay": (lambda: graph.replay() or 1, [])}
        for _ in range(2):   # warm-up
            for f, _ in ways.values():
                f()
        for _ in range(a.rounds):
            for name, (f, res) in ways.items():
                res.append(timed(f, a.seconds))
        for name, (f, res) in ways.items():
            row = {"workload": "model(x) 1x17", "size": "256x256", "way": name}
            for k in res[0]:
                row[k] = sum(r[k] for r in res) / len(res)
            out["rows"].append(row)
            print(json.dumps(row), flush=True)
    out["card_after"] = card()
    print(json.dumps(out["card_after"]), flush=True)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
