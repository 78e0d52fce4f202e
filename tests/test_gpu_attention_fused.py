"""The fused per-frame attention kernel (attn_tc.cu): frames of more than 32 x 32 latent positions run softmax(Q K^T / sqrt(C))
V with an online softmax on wgmma, without the tokens x tokens score matrix.

GPU checks: op-level accuracy against fp64 SDPA (diffuse inputs, and inputs whose row maxima sit in the last KV tile so
that the running-max rescale is exercised), a 2160 x 3840 frame (270 x 480 latents), launch lists on both sides of the
1024-token threshold, frame independence, a 1080p stream of kl_causal_488_4chn and parity of reduced-width causal models
with the CPU oracle at a latent frame of 33 x 34.  CPU check: the kernel's MMAs are pipelined in the compiled library."""
import ctypes as C
import json
import math
import os
import sys

import pytest
import torch

from vidtok_b200 import _native as N

X3_TOL = 4e-5        # EXACT_TC op gate (tests/test_gpu_ops_tc.py)
BF16_TOL = 3e-2      # BF16 attention gate (test_attention_core_wgmma)
PRECS = [N.PREC_BF16, N.PREC_EXACT_TC]
PIDS = ["bf16", "exact_tc"]
gpu = pytest.mark.gpu


def _p(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _to_act(x, precision):
    """fp32 [frames, tokens, C] cuda -> the precision's activation rows (bf16, or hi|lo fp16 planes)"""
    if precision == N.PREC_BF16:
        return x.to(torch.bfloat16).contiguous()
    hi = x.clamp(-65504.0, 65504.0).to(torch.float16)
    lo = (x - hi.float()).clamp(-65504.0, 65504.0).to(torch.float16)
    return torch.cat([hi, lo], dim=-1).contiguous()


def _from_act(y, precision):
    if precision == N.PREC_BF16:
        return y.float()
    c = y.shape[-1] // 2
    return y[..., :c].float() + y[..., c:].float()


def _operands(frames, tokens, C_, seed, peaked):
    """q, k, v fp32 on the device.  peaked: a shared direction u (|u| = sqrt(C)) added to every query, and 20 u / sqrt(C) to
    the last token's key, so that every row's maximum lies in the last KV tile (that score rises by 10 over the others)"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    q, k, v = (torch.randn(frames, tokens, C_, generator=g, device="cuda") for _ in range(3))
    if peaked:
        u = torch.randn(C_, generator=g, device="cuda")
        u = u / u.norm() * math.sqrt(C_)
        q += 0.5 * u
        k[:, -1] += 20.0 * u / math.sqrt(C_)
    return q, k, v


def _attention(precision, qa, ka, va, frames, H, W, C_, profile=False, ws_bytes=None):
    o = torch.empty_like(qa)
    if ws_bytes is None:
        ws_bytes = 3 * qa.numel() * qa.element_size() + (1 << 20)   # output + V^T + slack: no tokens x tokens term
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    lib = N.lib()
    if profile:
        lib.vt_profile_start()
    N.check(lib.vt_op_attention_hw(precision, _p(qa), _p(ka), _p(va), _p(o), frames, H, W, C_, _p(ws), ws.numel(), _stream()))
    torch.cuda.synchronize()
    names = {}
    if profile:
        buf = C.create_string_buffer(1 << 16)
        n = lib.vt_profile_stop(buf, len(buf))
        names = {k_: v_["launches"] for k_, v_ in json.loads(buf.value.decode()).items()} if n > 0 else {}
    return o, names


def _ref_rows(q, k, v, rows):
    """fp64 SDPA of the query rows `rows` (one frame), on the device in blocks"""
    out = []
    kd, vd = k.double(), v.double()
    scale = 1.0 / math.sqrt(q.shape[-1])
    for i in range(0, len(rows), 1024):
        r = rows[i:i + 1024]
        s = (q[r].double() @ kd.T) * scale
        out.append(torch.softmax(s, dim=-1) @ vd)
    return torch.cat(out)


def _sample_rows(tokens, seed=0):
    """the first, a middle and the last 64-row query tile, and 512 rows at random"""
    mid = (tokens // 2) // 64 * 64
    last = (tokens - 1) // 64 * 64
    rows = set(range(0, 64)) | set(range(mid, mid + 64)) | set(range(last, tokens))
    g = torch.Generator().manual_seed(seed)
    rows |= set(torch.randint(0, tokens, (512,), generator=g).tolist())
    return torch.tensor(sorted(rows), device="cuda")


def _check(precision, H, W, peaked, full, C_=512, frames=1, seed=1):
    tokens = H * W
    q, k, v = _operands(frames, tokens, C_, seed, peaked)
    qa, ka, va = (_to_act(t, precision) for t in (q, k, v))
    qs, ks, vs = (_from_act(t, precision) for t in (qa, ka, va))    # the values the kernel sees
    o, names = _attention(precision, qa, ka, va, frames, H, W, C_, profile=True)
    assert names.get("attn_tc3" if precision == N.PREC_EXACT_TC else "attn_tc", 0) == 1, names
    got = _from_act(o, precision)
    worst = 0.0
    for f in range(frames):
        rows = torch.arange(tokens, device="cuda") if full else _sample_rows(tokens, seed=f)
        ref = _ref_rows(qs[f], ks[f], vs[f], rows)
        worst = max(worst, float((got[f][rows].double() - ref).abs().max()))
    tol = BF16_TOL if precision == N.PREC_BF16 else X3_TOL
    print(f"[attn_tc {H}x{W} prec {precision} peaked={peaked}] max err {worst:.3e}")
    assert worst <= tol, f"{H}x{W} peaked={peaked}: max err {worst:.3e} > {tol}"
    return worst


@gpu
@pytest.mark.parametrize("peaked", [False, True], ids=["diffuse", "peaked"])
@pytest.mark.parametrize("precision", PRECS, ids=PIDS)
@pytest.mark.parametrize("hw", [(33, 33), (45, 80), (90, 160), (135, 240)], ids=lambda t: f"{t[0]}x{t[1]}")
def test_fused_attention_vs_fp64(hw, precision, peaked):
    """33 x 33 (1 089 tokens: a 1-row last query tile), 45 x 80, 90 x 160 and one 135 x 240 frame; every row up to 45 x 80,
    sampled query tiles above (the rows are independent)"""
    H, W = hw
    _check(precision, H, W, peaked, full=H * W <= 3600)


@gpu
@pytest.mark.parametrize("precision", PRECS, ids=PIDS)
def test_fused_attention_4k_frame(precision):
    """one 2160 x 3840 frame (270 x 480 = 129 600 tokens): it runs in a workspace of the output and V^T alone (the score
    matrix would be 67 GB) and matches fp64 on the first, a middle and the last query tile"""
    _check(precision, 270, 480, False, full=False)


@gpu
def test_launch_lists_around_the_threshold():
    C_ = 512
    for precision in PRECS:
        fused = "attn_tc3" if precision == N.PREC_EXACT_TC else "attn_tc"
        q, k, v = _operands(2, 48 * 48, C_, 3, False)
        _, names = _attention(precision, *(_to_act(t, precision) for t in (q, k, v)), 2, 48, 48, C_, profile=True)
        assert names.get(fused, 0) == 1, names
        assert not any(n.startswith(("gemm_simt", "softmax_rows", "conv_tc")) for n in names), names
        # 32 x 32: the two-GEMM path, unchanged
        q, k, v = _operands(2, 32 * 32, C_, 3, False)
        _, names = _attention(precision, *(_to_act(t, precision) for t in (q, k, v)), 2, 32, 32, C_, profile=True,
                              ws_bytes=2 * 1024 * (8 * 1024 + 24 * C_) + 65536)
        assert not any(n.startswith("attn_") for n in names), names
        assert names.get("conv_tc3" if precision == N.PREC_EXACT_TC else "conv_tc", 0) == 2, names


@gpu
@pytest.mark.parametrize("precision", PRECS, ids=PIDS)
def test_frames_are_independent(precision):
    """a 3-frame launch equals three 1-frame launches bit for bit, and a frame gives the same bits at another index of
    another launch"""
    H, W, C_ = 33, 40, 512
    q, k, v = (_to_act(t, precision) for t in _operands(3, H * W, C_, 5, False))
    o3, _ = _attention(precision, q, k, v, 3, H, W, C_)
    for f in range(3):
        o1, _ = _attention(precision, q[f:f + 1].contiguous(), k[f:f + 1].contiguous(), v[f:f + 1].contiguous(), 1, H, W, C_)
        assert torch.equal(o1[0], o3[f]), f
    perm = [2, 0, 1]
    o3p, _ = _attention(precision, q[perm].contiguous(), k[perm].contiguous(), v[perm].contiguous(), 3, H, W, C_)
    for i, f in enumerate(perm):
        assert torch.equal(o3p[i], o3[f]), (i, f)


def _kl488():
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
    from oracle.make_golden import model_yaml
    from vidtok_b200.compat_util import instantiate_from_config
    from vidtok_b200.synth import synth_state_dict
    cfg = model_yaml(version="v1_0", reg="kl", ch=128, ch_mult=(1, 2, 4, 4), z=4, interp=None)
    cfg["params"]["decoder_config"]["params"] = dict(cfg["params"]["encoder_config"]["params"])
    cfg["params"]["regularizer_config"]["params"] = {"sample": False}
    model = instantiate_from_config(cfg)
    model.load_state_dict(synth_state_dict({k: tuple(v.shape) for k, v in model.state_dict().items()}, seed=0))
    return model.cuda().eval()


def _launches(fn):
    lib = N.lib()
    lib.vt_profile_start()
    out = fn()
    torch.cuda.synchronize()
    buf = C.create_string_buffer(1 << 16)
    n = lib.vt_profile_stop(buf, len(buf))
    prof = json.loads(buf.value.decode()) if n > 0 else {}
    return out, {k: v["launches"] for k, v in prof.items()}


@gpu
def test_kl488_1080p_bf16_stream():
    """kl_causal_488_4chn (synthetic weights), 1080 x 1920 bf16: a stream of 1 + 4 frames equals the whole 5-frame clip bit
    for bit and runs the fused attention (no FMA GEMM).  A 4-frame chunk's workspace grows from 720p to 1080p with the
    pixel count (x 2.25), with no term in tokens^2 (the materialised attention would add 6.3 GB at 1080p)"""
    from vidtok_b200.streaming import EncodeStream
    from vidtok_b200.synth import synth_clip
    model = _kl488()
    model.precision = "bf16"
    x = synth_clip(1, 5, 1080, 1920, seed=11).cuda()
    with torch.no_grad():
        z_w, lw = _launches(lambda: model.encode(x))
        enc720 = EncodeStream(model, 1, 720, 1280)
        ws720 = N.lib().vt_chunk_workspace_bytes(enc720.state.handle, 4)
        enc720.close()
        enc = EncodeStream(model, 1, 1080, 1920)
        ws4 = N.lib().vt_chunk_workspace_bytes(enc.state.handle, 4)

        def stream():
            z0, _ = enc.push(x[:, :, :1])
            z1, _ = enc.push(x[:, :, 1:5])
            return torch.cat([z0, z1], dim=2)
        z_s, ls = _launches(stream)
        enc.close()
    assert torch.equal(z_s, z_w)
    for names in (lw, ls):
        assert names.get("attn_tc", 0) > 0 and "gemm_simt" not in names and "softmax_rows" not in names, names
    print(f"[1080p bf16] chunk workspace (4 frames) {ws4 / 1e9:.2f} GB, 720p {ws720 / 1e9:.2f} GB")
    assert 0 < ws4 <= 2.25 * 1.02 * ws720, (ws4, ws720)


def _reduced_cfg(reg, z):
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
    from oracle.make_golden import model_yaml
    cfg = model_yaml(version="v1_0", reg=reg, ch=64, ch_mult=(1, 2, 4, 4), z=z, interp=None)
    cfg["params"]["decoder_config"]["params"] = dict(cfg["params"]["encoder_config"]["params"])
    if reg == "kl":
        cfg["params"]["regularizer_config"]["params"] = {"sample": False}
    return cfg


@gpu
@pytest.mark.parametrize("reg", ["kl", "fsq"])
def test_parity_with_oracle_above_threshold(reg):
    """causal v1.0 models of width 64 (mid C = 256), 5 x 264 x 272 frames: the mid attention blocks see 33 x 34 = 1 122
    tokens (above the threshold, not a multiple of 64).  exact mode within the 1e-3 latent / reconstruction gate of the
    oracle; FSQ codes equal outside the 1e-4 tie band"""
    from oracle.vidtok_oracle import OracleModel, cfg_from_model_yaml
    from vidtok_b200.compat_util import instantiate_from_config
    from vidtok_b200.synth import synth_clip, synth_state_dict
    cfg = _reduced_cfg(reg, 4 if reg == "kl" else 5)
    model = instantiate_from_config(cfg)
    sd = synth_state_dict({k: tuple(v.shape) for k, v in model.state_dict().items()}, seed=2)
    model.load_state_dict(sd)
    model = model.cuda().eval()
    model.precision = "exact"
    x = synth_clip(1, 5, 264, 272, seed=13)
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    om = OracleModel(cfg_from_model_yaml(cfg), sd)
    with torch.no_grad():
        if reg == "kl":
            z_o, dec_o, _ = om.forward(x)
            (z, dec, _), names = _launches(lambda: model(x.cuda()))
            dz, dd = float((z.cpu() - z_o).abs().max()), float((dec.cpu() - dec_o).abs().max())
            print(f"[parity kl 33x34] max|dz|={dz:.2e} max|ddec|={dd:.2e}")
            assert dz <= 1e-3 and dd <= 1e-3
        else:
            _, log_o, _ = om.encode(x, return_pre=True)
            (_, log), names = _launches(lambda: model.encode(x.cuda(), return_reg_log=True))
            idx = log["indices"].cpu()
            bad = idx != log_o["indices"]
            pre = log_o["pre_round"]
            near = ((pre - pre.floor() - 0.5).abs() < 1e-4).any(dim=-1)
            print(f"[parity fsq 33x34] raw mismatches {int(bad.sum())}/{bad.numel()}")
            assert not (bad & ~near).any()
    assert names.get("attn_tc3", 0) > 0 and "gemm_simt" not in names, names


def test_fused_attention_kernel_is_pipelined():
    """the fused attention's bf16 and split instantiations issue HGMMA and keep more than one in flight"""
    from vidtok_b200 import build, sass
    lib = build.build()
    kernels = sass.kernel_counts(sass.disassemble(lib))
    hg = {name: k for name, k in kernels.items() if k.get("HGMMA", 0) > 0}
    for want in ("attn_tc_kernelILb0E", "attn_tc_kernelILb1E"):
        assert any(want in n for n in hg), f"no HGMMA in {want}"
    mine = {n: k for n, k in hg.items() if "attn_tc_kernel" in n}
    assert not sass.serialized_wgmma_kernels(mine), sorted(sass.demangle(mine))
