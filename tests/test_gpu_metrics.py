"""-m gpu: the fused per-frame PSNR / SSIM (vidtok_b200.metrics) against compat_util.compute_psnr / compute_ssim evaluated
frame by frame in float64 on the CPU on (clamp(v, -1, 1) + 1) / 2 (tests/test_dropin_scripts.py pins those two functions to
the reference's formulas).  Inputs are seeded and made here: a smooth random field plus noise for x, y = x + noise with a
share of the values pushed outside [-1, 1] so that the clamp matters.

Tolerances: the largest deviations from float64 seen on an H100 over every case below were 9.8e-7 dB (PSNR) and 4.5e-7
(SSIM; the 11 x 11 frame whose map is one position, 6.3e-8 elsewhere), against 3.4e-6 dB and 6.0e-6 for compat_util's own
fp32 CUDA result; the bounds are about five times what was seen.  Each test prints what it saw."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from conftest import load_golden, resolved_model_cfg, synth_weights  # noqa: E402
from vidtok_b200 import _native as N  # noqa: E402
from vidtok_b200.compat_util import compute_psnr, compute_ssim  # noqa: E402
from vidtok_b200.metrics import Scorer, frame_scores  # noqa: E402

PSNR_TOL, SSIM_TOL = 5e-6, 2e-6


def make_pair(shape, seed, strength):
    g = torch.Generator().manual_seed(seed)
    lead, (H, W) = shape[:-2], shape[-2:]
    n = math.prod(lead)
    coarse = torch.randn((n, 1, max(2, H // 16), max(2, W // 16)), generator=g)
    x = F.interpolate(coarse, size=(H, W), mode="bilinear", align_corners=False).reshape(shape) * 0.6
    x = (x + 0.05 * torch.randn(shape, generator=g)).clamp(-1, 1)
    y = x + strength * torch.randn(shape, generator=g)
    push = torch.rand(shape, generator=g) < 0.02
    y = torch.where(push, y * 4.0, y)
    return x.contiguous(), y.contiguous()


def as_frames(t):
    return t.permute(0, 2, 1, 3, 4).reshape(-1, t.shape[1], t.shape[3], t.shape[4]) if t.dim() == 5 else t


def reference(x, y, dtype=torch.float64, device="cpu", ssim=True):
    """per-frame (psnr, ssim) of compat_util on the script's preprocessing, as float64 CPU tensors"""
    a = (as_frames(x).to(device, dtype).clamp(-1, 1) + 1) / 2
    b = (as_frames(y).to(device, dtype).clamp(-1, 1) + 1) / 2
    ps = torch.stack([compute_psnr(a[i:i + 1], b[i:i + 1]) for i in range(a.shape[0])])
    ss = torch.stack([compute_ssim(a[i:i + 1], b[i:i + 1]) for i in range(a.shape[0])]) if ssim else ps
    return ps.double().cpu(), ss.double().cpu()


def errors(got, want):
    return float((got.double().cpu().reshape(-1) - want).abs().max())


# (id, shape): clips [B,C,T,H,W] and one batch of frames [N,C,H,W]
CASES = [
    ("kl488_batch", (8, 3, 17, 256, 256)),
    ("128", (2, 3, 5, 128, 128)),
    ("240x360_tile_remainders", (1, 3, 4, 240, 360)),
    ("11x11_one_position", (1, 3, 2, 11, 11)),
    ("21x300", (1, 3, 2, 21, 300)),
    ("one_channel", (1, 1, 3, 256, 256)),
    ("640_tie_f2", (1, 3, 2, 640, 640)),
    ("720p_f3_drops_a_column", (1, 3, 2, 720, 1280)),
    ("1080p_f4", (1, 3, 2, 1080, 1920)),
    ("odd_width_f2_scalar", (1, 2, 2, 531, 643)),
    ("frames_4d", (32, 3, 256, 256)),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_frame_scores_match_float64_reference(case):
    name, shape = case
    worst_p = worst_s = 0.0
    for k, strength in enumerate((0.01, 0.08, 0.4)):
        if k > 0 and math.prod(shape) > 3e7:       # the large batches take one strength: the CPU reference is the slow part
            break
        x, y = make_pair(shape, seed=1000 * len(shape) + 7 * k + shape[-1], strength=strength)
        ps, ss = frame_scores(x.cuda(), y.cuda())
        assert ps.dtype == torch.float32 and tuple(ps.shape) == ((shape[0], shape[2]) if len(shape) == 5 else (shape[0],))
        assert ss.shape == ps.shape
        rp, rs = reference(x, y)
        ep, es = errors(ps, rp), errors(ss, rs)
        worst_p, worst_s = max(worst_p, ep), max(worst_s, es)
        if math.prod(shape) <= 3e7:
            # compat_util's own fp32 result on the device is the accuracy the fused kernel replaces
            cp, cs = reference(x, y, torch.float32, "cuda")
            cep, ces = errors(cp, rp), errors(cs, rs)
            print(f"{name} s={strength}: fused |dPSNR| {ep:.2e} |dSSIM| {es:.2e}; torch fp32 {cep:.2e} {ces:.2e}")
            assert ep <= max(2 * cep, PSNR_TOL) and es <= max(2 * ces, SSIM_TOL)
    print(f"{name}: max |dPSNR| {worst_p:.3g} dB, max |dSSIM| {worst_s:.3g}")
    assert worst_p <= PSNR_TOL and worst_s <= SSIM_TOL


def test_half_precision_inputs_equal_their_float_values_bit_for_bit():
    x, y = make_pair((2, 3, 3, 96, 136), seed=5, strength=0.1)
    x, y = x.cuda(), y.cuda()
    for dt in (torch.bfloat16, torch.float16):
        yl, xl = y.to(dt), x.to(dt)
        want = frame_scores(x, yl.float())
        got = frame_scores(x, yl)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]), dt
        want = frame_scores(xl.float(), yl.float())
        got = frame_scores(xl, yl)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]), dt
    # an odd width takes the element-wise loads
    x, y = make_pair((1, 3, 2, 40, 51), seed=6, strength=0.1)
    got, want = frame_scores(x.cuda(), y.cuda().bfloat16()), frame_scores(x.cuda(), y.bfloat16().float().cuda())
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


@pytest.mark.parametrize("shape", [(1, 3, 2, 256, 256), (1, 3, 2, 100, 75), (1, 3, 1, 720, 1280)])
def test_equal_clips_score_exactly(shape):
    top = torch.tensor(-10.0 * math.log10(1e-8), dtype=torch.float32)
    x, _ = make_pair(shape, seed=9, strength=0.0)
    for clip in (x.cuda() * 1.5, torch.zeros(shape, device="cuda")):     # * 1.5: some values beyond the clamp
        ps, ss = frame_scores(clip, clip.clone())
        assert torch.all(ss == 1.0), ss
        assert torch.all(ps.cpu() == top), ps


def test_deterministic_and_stream_independent():
    x, y = make_pair((2, 3, 4, 240, 360), seed=11, strength=0.1)
    x, y = x.cuda(), y.cuda()
    a = frame_scores(x, y)
    b = frame_scores(x, y)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        c = frame_scores(x, y)
    side.synchronize()
    assert torch.equal(a[0], c[0]) and torch.equal(a[1], c[1])


def test_psnr_only():
    x, y = make_pair((2, 3, 3, 240, 360), seed=12, strength=0.1)
    both = frame_scores(x.cuda(), y.cuda())
    ps, none = frame_scores(x.cuda(), y.cuda(), ssim=False)
    assert none is None and torch.equal(ps, both[0])
    # frames too small for an SSIM window still have a PSNR
    x, y = make_pair((1, 3, 2, 7, 9), seed=13, strength=0.1)
    ps, _ = frame_scores(x.cuda(), y.cuda(), ssim=False)
    assert errors(ps, reference(x, y, ssim=False)[0]) <= PSNR_TOL
    # the ABI writes nothing through a null ssim pointer and leaves running[1] alone
    xs, ys = x.cuda(), y.cuda()
    running = torch.zeros(3, dtype=torch.float64, device="cuda")
    out = torch.empty(2, device="cuda")
    ws = torch.empty(N.lib().vt_frame_scores_workspace_bytes(1, 3, 2, 7, 9), dtype=torch.uint8, device="cuda")
    rc = N.lib().vt_frame_scores(C.c_void_p(xs.data_ptr()), 0, C.c_void_p(ys.data_ptr()), 0, 1, 3, 2, 7, 9, C.c_void_p(out.data_ptr()), None,
                                 C.c_void_p(running.data_ptr()), C.c_void_p(ws.data_ptr()), ws.numel(),
                                 C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0
    assert torch.equal(out, ps.reshape(-1)) and running.tolist() == [float(out.double().sum()), 0.0, 2.0]


def test_scorer_accumulates_without_synchronising():
    x, y = make_pair((1, 3, 17, 128, 160), seed=14, strength=0.08)
    x, y = x.cuda(), y.cuda()
    whole = Scorer()
    ps, ss = whole.update(x, y)
    pieces = Scorer()
    t0 = 0
    for n in (4, 4, 4, 5):
        pieces.update(x[:, :, t0:t0 + n], y[:, :, t0:t0 + n])
        t0 += n
    a, b = whole.sums().cpu(), pieces.sums().cpu()
    assert float(((a - b).abs() / a.abs()).max()) <= 1e-12, (a, b)
    r = pieces.result()
    assert r["frames"] == 17
    assert abs(r["psnr"] - float(ps.double().mean())) <= 1e-12 * abs(r["psnr"])
    assert abs(r["ssim"] - float(ss.double().mean())) <= 1e-12
    assert pieces.result(reduce=False) == r
    rp, rs = reference(x.cpu(), y.cpu())
    assert abs(r["psnr"] - float(rp.mean())) <= PSNR_TOL and abs(r["ssim"] - float(rs.mean())) <= SSIM_TOL
    # the evaluation script's number: groups of 16 frames, each group's value once per frame
    a01, b01 = (as_frames(x.cpu()).double().clamp(-1, 1) + 1) / 2, (as_frames(y.cpu()).double().clamp(-1, 1) + 1) / 2
    script = []
    for u, v in zip(torch.split(a01, 16), torch.split(b01, 16)):
        script += [compute_ssim(u, v).item()] * u.shape[0]
    assert abs(r["ssim"] - sum(script) / len(script)) <= SSIM_TOL
    pieces.reset()
    assert pieces.result()["frames"] == 0

    # an update at a geometry the scorer has seen enqueues work and nothing else
    whole.update(x, y)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        whole.update(x, y)
        whole.update(x[:, :, :4].contiguous(), y[:, :, :4].contiguous())
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert whole.result()["frames"] == 17 * 3 + 4


def test_dist_partials_on_one_rank():
    from vidtok_b200 import dist
    x, y = make_pair((2, 3, 3, 64, 64), seed=15, strength=0.1)
    part = dist.score_partial(x.cuda(), y.cuda())
    assert part.dtype == torch.float64 and tuple(part.shape) == (3,)
    ps, ss = frame_scores(x.cuda(), y.cuda())
    r = dist.global_scores(part)
    assert r["frames"] == 6 and abs(r["psnr"] - float(ps.double().mean())) <= 1e-12 * r["psnr"] and abs(r["ssim"] - float(ss.double().mean())) <= 1e-12


def test_abi_errors_launch_nothing():
    L = N.lib()
    x = torch.zeros((1, 3, 2, 32, 32), device="cuda")
    ps, ss = torch.empty(2, device="cuda"), torch.empty(2, device="cuda")
    ws = torch.empty(L.vt_frame_scores_workspace_bytes(1, 3, 2, 32, 32), dtype=torch.uint8, device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr())   # noqa: E731
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    L.vt_launch_count(1)
    assert L.vt_frame_scores(None, 0, p(x), 0, 1, 3, 2, 32, 32, p(ps), p(ss), None, p(ws), ws.numel(), s) == -1
    assert b"null argument" in L.vt_last_error()
    assert L.vt_frame_scores(p(x), 0, p(x), 0, 1, 3, 2, 32, 32, None, p(ss), None, p(ws), ws.numel(), s) == -1
    assert L.vt_frame_scores(p(x), 0, p(x), 0, 1, 3, 2, 32, 32, p(ps), p(ss), None, None, ws.numel(), s) == -1
    assert L.vt_frame_scores(p(x), 3, p(x), 0, 1, 3, 2, 32, 32, p(ps), p(ss), None, p(ws), ws.numel(), s) == -1
    assert b"unknown dtype" in L.vt_last_error()
    assert L.vt_frame_scores(p(x), 0, p(x), -1, 1, 3, 2, 32, 32, p(ps), p(ss), None, p(ws), ws.numel(), s) == -1
    assert L.vt_frame_scores(p(x), 0, p(x), 0, 1, 3, 0, 32, 32, p(ps), p(ss), None, p(ws), ws.numel(), s) == -1
    assert L.vt_frame_scores(p(x), 0, p(x), 0, 1, 3, 2, 10, 64, p(ps), p(ss), None, p(ws), ws.numel(), s) == -1
    assert b"Input size: 10 x 64" in L.vt_last_error()
    assert L.vt_frame_scores(p(x), 0, p(x), 0, 1, 3, 2, 32, 32, p(ps), p(ss), None, p(ws), ws.numel() - 1, s) == -4
    assert b"workspace too small" in L.vt_last_error()
    assert L.vt_launch_count(0) == 0
    assert L.vt_frame_scores(p(x), 0, p(x), 0, 1, 3, 2, 32, 32, p(ps), p(ss), None, p(ws), ws.numel(), s) == 0
    assert L.vt_launch_count(0) == 2
    torch.cuda.synchronize()
    x4 = torch.zeros((2, 3, 10, 64), device="cuda")
    with pytest.raises(ValueError, match="Input size: 10 x 64"):
        frame_scores(x4, x4)


def test_scores_a_model_and_a_decode_stream():
    from vidtok_b200.compat_util import instantiate_from_config
    from vidtok_b200.streaming import DecodeStream
    from vidtok_b200.synth import synth_clip
    d, meta = load_golden("tiny_kl_v10")
    model = instantiate_from_config(resolved_model_cfg(meta))
    missing, unexpected = model.load_state_dict(synth_weights(meta, d), strict=False)
    assert not missing and not unexpected
    model = model.to("cuda").eval()
    B, _, T, H, W = meta["input"]
    x = synth_clip(B, T, H, W, seed=meta["input_seed"]).cuda()
    with torch.no_grad():
        torch.manual_seed(1)
        z, recon, _ = model(x)
        scorer = Scorer()
        scorer.update(x, recon)
        got = scorer.result()
        rp, rs = reference(x.cpu(), recon.cpu())
        print(f"forward: PSNR {got['psnr']:.4f} SSIM {got['ssim']:.5f} over {got['frames']} frames")
        assert got["frames"] == B * T
        assert abs(got["psnr"] - float(rp.mean())) <= PSNR_TOL and abs(got["ssim"] - float(rs.mean())) <= SSIM_TOL

        # the same video decoded in pushes, scored push by push
        dec = DecodeStream(model, B, z.shape[3], z.shape[4])
        scorer.reset()
        outs, t0 = [], 0
        for zs in (z[:, :, :2], z[:, :, 2:]):
            out = dec.push(zs)
            scorer.update(x[:, :, t0:t0 + out.shape[2]], out)
            outs.append(out)
            t0 += out.shape[2]
        dec.close()
        assert t0 == T
        got = scorer.result()
        rp, rs = reference(x.cpu(), torch.cat(outs, dim=2).cpu())
        assert got["frames"] == B * T
        assert abs(got["psnr"] - float(rp.mean())) <= PSNR_TOL and abs(got["ssim"] - float(rs.mean())) <= SSIM_TOL
