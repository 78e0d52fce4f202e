"""Per-frame time of the attention core (vt_op_attention_hw) at C = 512 in bf16 and exact, for frames of 32x32 .. 270x480
latent positions, with the achieved rate from the algorithmic 4 tokens^2 C FLOPs per frame.  Each point is timed with CUDA
events over at least 0.5 s after a warm-up call.  Shapes a build cannot run (workspace beyond the card) are reported as such.

With several --lib arguments the libraries are measured alternately, each in its own process, --rounds times (the same
session, the same card), so that two builds can be compared.  Prints one JSON line per point and the card, its power limit
and SM clocks.
usage: python tools/bench_attention.py [--lib PATH ...] [--rounds 2] [--out FILE]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FRAMES = [(32, 32), (48, 48), (45, 80), (90, 160), (135, 240), (180, 320), (270, 480)]
C_ = 512


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:
        return f"(nvidia-smi unavailable: {e})"


def child(lib_path, tag):
    import torch
    sys.path.insert(0, ROOT)
    from vidtok_b200 import _native as N
    if lib_path:
        N.LIB_PATH = os.path.abspath(lib_path)
    lib = N.lib()
    if not torch.cuda.is_available():
        raise SystemExit("bench_attention: no CUDA device; these numbers need an H100")
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    free = torch.cuda.mem_get_info()[0]
    for prec, name in ((N.PREC_BF16, "bf16"), (N.PREC_EXACT_TC, "exact")):
        cw = 2 if prec == N.PREC_EXACT_TC else 1
        dt = torch.float16 if cw == 2 else torch.bfloat16
        for H, W in FRAMES:
            tokens = H * W
            row = {"lib": tag, "precision": name, "frame": f"{H}x{W}", "tokens": tokens}
            act = tokens * C_ * cw * 2
            # the two-GEMM path needs S (fp32) + P (2 or 4 B) + V^T per frame; the fused path V^T; give either what it asks
            ws_bytes = tokens * tokens * (4 + 2 * cw) + 2 * act + (64 << 20)
            if 4 * act + ws_bytes > 0.9 * free:
                ws_bytes = 2 * act + (64 << 20)
            try:
                q, k, v = (torch.randn(tokens, C_ * cw, device="cuda").to(dt) for _ in range(3))
                o = torch.empty_like(q)
                ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
            except torch.cuda.OutOfMemoryError:
                row["result"] = "does not fit on the card"
                print(json.dumps(row), flush=True)
                continue

            def call():
                return lib.vt_op_attention_hw(prec, C.c_void_p(q.data_ptr()), C.c_void_p(k.data_ptr()), C.c_void_p(v.data_ptr()),
                                              C.c_void_p(o.data_ptr()), 1, H, W, C_, C.c_void_p(ws.data_ptr()), ws.numel(), s)
            rc = call()
            torch.cuda.synchronize()
            if rc != 0:
                row["result"] = "cannot run: " + lib.vt_last_error().decode(errors="replace")
                print(json.dumps(row), flush=True)
                del q, k, v, o, ws
                torch.cuda.empty_cache()
                continue
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            n, ms = 1, 0.0
            while True:
                a.record()
                for _ in range(n):
                    call()
                b.record()
                torch.cuda.synchronize()
                ms = a.elapsed_time(b)
                if ms >= 500.0:
                    break
                n = max(n * 2, int(n * 550.0 / max(ms, 1e-3)) + 1)
            per = ms / n
            row.update({"calls": n, "ms_per_frame": round(per, 4), "TFLOP_per_s": round(4.0 * tokens * tokens * C_ / (per * 1e-3) / 1e12, 1)})
            print(json.dumps(row), flush=True)
            del q, k, v, o, ws
            torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=None, help="library to measure (default: the in-tree build)")
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child is not None:
        child(args.child, args.child or "in-tree")
        return
    libs = args.lib or [""]
    rows = []
    before = card()
    for r in range(args.rounds):
        for lp in libs:
            out = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", lp], capture_output=True, text=True)
            if out.returncode != 0:
                raise SystemExit(f"bench_attention child {lp or 'in-tree'} failed:\n{out.stderr[-4000:]}")
            for line in out.stdout.splitlines():
                if line.startswith("{"):
                    d = json.loads(line)
                    d["round"] = r
                    rows.append(d)
                    print(json.dumps(d), flush=True)
    res = {"card_before": before, "card_after": card(), "C": C_, "rows": rows}
    print(json.dumps({"card_before": res["card_before"], "card_after": res["card_after"]}))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
