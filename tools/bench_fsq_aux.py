"""Times the FSQ aux loss on the device (csrc/fsq_aux.cu) and what it costs the fsq488 forward.

  python tools/bench_fsq_aux.py [--out DIR]

1. the aux kernels alone (partials + finalize of one segment) at 40 960 tokens (the fsq488 batch: 8 clips 17x256x256 ->
   5x32x32 latents) for 4, 5 and 6 digits of 8 levels, with peaked and flat latents: CUDA events around many launches;
2. the fsq488 forward (mixed precision, as bench.py runs it) with the shipped weights against the same model with both weights
   0, alternated in one process, median of 3 rounds;
3. the materialised fp32 form of the reference (regularizers.py:234-239: tokens x codebook distance, softmax, entropy, mean)
   on the GPU at B = 1 and B = 8 for 32 768 codes: time and peak memory, or the out-of-memory error.
The card name and power limit are read in the same run.  Prints one JSON object (also written to DIR/bench_fsq_aux.json
with --out DIR)."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def latent(kind, d, seed):
    z = torch.randn((8, d, 5, 32, 32), generator=torch.Generator().manual_seed(seed))
    return (z * {"peaked": 2.5, "flat": 2e-3}[kind]).cuda()


def time_kernels(reps=20):
    from vidtok_b200.engine import FSQRegularizer
    out = []
    for d in (4, 5, 6):
        reg = FSQRegularizer([8] * d, entropy_loss_weight=0.1, entropy_loss_annealing_steps=2000, entropy_loss_annealing_factor=3,
                             commitment_loss_weight=0.25).cuda()
        for kind in ("peaked", "flat"):
            h = latent(kind, d, 10 + d)
            for _ in range(3):
                reg.aux_loss(h)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                reg.aux_loss(h)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / reps
            out.append({"digits": d, "codes": 8 ** d, "latent": kind, "tokens": 40960, "ms_per_call": round(ms, 4),
                        "aux_loss": float(reg.aux_loss(h))})
            print(f"[aux] {d} digits {kind:6s}: {ms:.3f} ms per partials + finalize", flush=True)
    return out


def time_forward(rounds=3, steps=3):
    import bench
    from vidtok_b200.compat_util import instantiate_from_config
    from vidtok_b200.synth import synth_clip, synth_state_dict
    cfg = bench.model_cfg(bench.CONFIGS["fsq488"])
    model = instantiate_from_config(cfg)
    model.load_state_dict(synth_state_dict({k: tuple(v.shape) for k, v in model.state_dict().items()}, seed=0))
    model = model.cuda().eval()
    model.precision = "mixed"
    reg = model.regularization
    shipped = (reg.entropy_loss_weight, reg.commitment_loss_weight)
    x = synth_clip(8, 17, 256, 256, seed=1234).cuda()

    def run(weights):
        reg.entropy_loss_weight, reg.commitment_loss_weight = weights
        with torch.no_grad():
            model(x)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(steps):
                model(x)
            torch.cuda.synchronize()
        return (time.perf_counter() - t0) / steps

    res = {"with_aux": [], "without_aux": []}
    for _ in range(rounds):
        res["with_aux"].append(run(shipped))
        res["without_aux"].append(run((0.0, 0.0)))
    reg.entropy_loss_weight, reg.commitment_loss_weight = shipped
    frames = 8 * 17
    out = {}
    for k, v in res.items():
        out[k] = {"step_s": [round(t, 4) for t in v], "median_step_s": round(statistics.median(v), 4),
                  "frames_per_s": round(frames / statistics.median(v), 2),
                  "spread_pct": round(100 * (max(v) - min(v)) / statistics.median(v), 2)}
    print(f"[fsq488] {json.dumps(out)}", flush=True)
    return out


def time_materialised():
    out = []
    J = 8 ** 5
    lv = torch.tensor([8] * 5, device="cuda")
    basis = torch.cumprod(torch.tensor([1, 8, 8, 8, 8], device="cuda"), 0)
    codebook = ((torch.arange(J, device="cuda")[:, None] // basis) % lv - 4).float() / 4
    for B in (1, 8):
        z = (torch.randn((B * 5 * 32 * 32, 5)) * 0.5).cuda()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.max_memory_allocated()
        try:
            t0 = time.perf_counter()
            prob = (2 * 100.0 * (z @ codebook.t())).softmax(dim=-1)
            ent = (-prob * prob.clamp(min=1e-5).log()).sum(-1).mean()
            avg = prob.mean(0)
            cbe = (-avg * avg.clamp(min=1e-5).log()).sum()
            float(ent - cbe)
            torch.cuda.synchronize()
            rec = {"B": B, "tokens": z.shape[0], "ms": round(1e3 * (time.perf_counter() - t0), 2),
                   "peak_growth_GiB": round((torch.cuda.max_memory_allocated() - base) / 2**30, 2)}
            del prob
        except torch.cuda.OutOfMemoryError as e:
            rec = {"B": B, "tokens": z.shape[0], "error": "out of memory: " + str(e).splitlines()[0][:160]}
        torch.cuda.empty_cache()
        print(f"[materialised] {rec}", flush=True)
        out.append(rec)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for bench_fsq_aux.json (default: print only)")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    import __graft_entry__ as ge
    ge.build()
    res = {"card_before": card(), "aux_kernels": time_kernels(), "fsq488_forward": time_forward(),
           "materialised_fp32_32768": time_materialised(), "card_after": card()}
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_fsq_aux.json"), "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
