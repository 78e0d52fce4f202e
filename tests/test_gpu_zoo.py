"""-m gpu: every tokenizer configuration the reference ships (the 23 YAMLs of tests/golden/zoo_manifest.json.gz), at the
width users load their checkpoints at (ch 128), on the device against float64.

bench.py runs four of these configurations and test_gpu_production_plans.py tests every kernel plan those four launch.
The rest of the zoo reaches code the four never do: the non-causal family's time padding (symmetric, and one zero frame
behind the end of the stride-2 time downsample, whose avg-pool window is shifted by one frame), its phase map of the
folded 2x time upsampling and its conv_stem padding; the KL epilogue at z = 8; the FSQ epilogue with 4 and 6 levels;
time downsampling x2 (288) and x8 (888 v1.1); spatial x4 (444: 64 x 64 latent frames through the fused attention); and
4x16x16 at 256 x 256 (16 x 16 latent frames).  Three tests close that gap:

  * test_zoo_model: one forward per YAML, seeded weights (synth_state_dict(seed=0)), a 1 x 3 x 17 x 256 x 256 clip (16
    frames for the non-causal family; each v1.1 YAML also tiled, chunk 16, over 33 frames), against OracleModel in float64
    on the device with the same noise.  Exact mode: latents and reconstruction within 1e-3 max-abs, FSQ indices equal
    outside the 1e-4 tie band, kl_loss within 1e-4 relative.  BF16 mode: the gates of test_gpu_model's
    test_bf16_mode_psnr_within_gate (PSNR within 0.01 dB, 0.05 dB for FSQ; KL reconstructions within 0.25 max-abs and
    0.02 mean-abs).
  * test_zoo_forward_keys_are_in_tables: the plan keys one bf16 and one exact forward of every YAML launch at the geometry
    above are all in PLAN_TABLE or ZOO_PLAN_TABLE, and no ZOO_PLAN_TABLE key is stale.
  * test_zoo_plan_case: every ZOO_PLAN_TABLE key through test_gpu_production_plans.run_case / check_case, with that
    module's bounds (bf16: 2^-7 |ref| + 2e-2; exact: 4e-5 (1 + |ref|); fp64 on the first kt-1, a middle and the last
    frame, where padding behind the end acts, and fp32 with TF32 off over the whole tensor).
"""
import gc
import gzip
import json
import os
import time

import pytest
import torch

pytestmark = pytest.mark.gpu

from test_gpu_production_plans import PLAN_TABLE, check_case, entry_of, parse, prec_of, run_case  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ZOO = json.load(gzip.open(os.path.join(ROOT, "tests", "golden", "zoo_manifest.json.gz"), "rt"))
H = W = 256
TILE_CHUNK, TILE_FRAMES = 16, 33
INPUT_SEED, NOISE_SEED = 1234, 4321
TOL = 1e-3
# (YAML, tiled): every YAML whole-clip, and the v1.1 ones again through tile_encode / tile_decode
MODEL_CASES = [(n, False) for n in sorted(ZOO)] + [(n, True) for n in sorted(ZOO) if n.startswith("vidtok_v1_1/")]


def case_id(case):
    name, tiled = case
    return name.replace("vidtok_v1_1/", "v11/").replace("vidtok_", "").replace(".yaml", "") + ("-tiled" if tiled else "")


@pytest.fixture(autouse=True)
def _free_between_cases():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
    gc.collect()                   # the models' native weights and workspaces go with their handles
    torch.cuda.empty_cache()


def clip_frames(name, tiled):
    return TILE_FRAMES if tiled else (17 if ZOO[name]["is_causal"] else 16)


def zoo_model(name, tiled):
    """(model on cuda, state dict, input clip [1,3,T,256,256] on the CPU)"""
    from vidtok_b200.compat_util import instantiate_from_config
    from vidtok_b200.synth import synth_clip, synth_state_dict
    rec = ZOO[name]
    model = instantiate_from_config(rec["model"])
    sd = synth_state_dict({k: tuple(v) for k, v in rec["shapes"].items()}, seed=0)
    missing, unexpected = model.load_state_dict(sd, strict=False)
    assert not missing and not unexpected
    model = model.cuda().eval()
    if tiled:
        model.use_tiling = True
        model.t_chunk_enc = TILE_CHUNK
        model.t_chunk_dec = TILE_CHUNK // model.encoder.time_downsample_factor
        model.use_overlap = True
    return model, sd, synth_clip(1, clip_frames(name, tiled), H, W, seed=INPUT_SEED)


def device_noise(shape):
    """the reference's torch.randn(mean.shape) on the CPU generator (distributions.py:17), as the engine draws it"""
    return torch.randn(shape).cuda()


def oracle_forward(name, tiled, sd, x):
    """OracleModel in float64 on the device -> (z, dec, log, oracle); dec trimmed to the input's frames like forward()"""
    from oracle.vidtok_oracle import OracleModel, cfg_from_model_yaml
    om = OracleModel(cfg_from_model_yaml(ZOO[name]["model"]), {k: v.cuda() for k, v in sd.items()}, dtype=torch.float64)
    if tiled:
        om.use_tiling, om.use_overlap = True, True
        om.t_chunk_enc = TILE_CHUNK
        om.t_chunk_dec = TILE_CHUNK // om.cfg.time_downsample_factor
    torch.manual_seed(NOISE_SEED)
    z, log = om.encode(x.cuda(), device_noise)
    dec = om.decode(z)
    return z, dec[:, :, -x.shape[2]:], log, om


def psnr01(x, y):
    from vidtok_b200.compat_util import compute_psnr
    return float(compute_psnr((x.clamp(-1, 1) + 1) / 2, (y.clamp(-1, 1) + 1) / 2))


@pytest.mark.parametrize("case", MODEL_CASES, ids=case_id)
def test_zoo_model(case):
    name, tiled = case
    cfg = ZOO[name]["model"]["params"]
    fsq = "FSQ" in cfg["regularizer_config"]["target"]
    model, sd, x = zoo_model(name, tiled)
    t0 = time.time()
    z_o, dec_oracle, log_o, om = oracle_forward(name, tiled, sd, x)
    torch.cuda.synchronize()
    t_oracle = time.time() - t0
    xd = x.cuda()
    fails = []

    # exact mode against the float64 oracle
    t0 = time.time()
    model.precision = "exact"
    with torch.no_grad():
        torch.manual_seed(NOISE_SEED)
        z, dec, log = model(xd)
    torch.cuda.synchronize()
    t_exact = time.time() - t0
    assert tuple(z.shape) == tuple(z_o.shape) and tuple(dec.shape) == tuple(dec_oracle.shape) == tuple(x.shape)
    msg = f"[{case_id(case)}] exact:"
    dec_o, zerr = dec_oracle, (z.double() - z_o).abs()
    if fsq:
        levels = tuple(cfg["regularizer_config"]["params"]["levels"])
        idx, idx_o, pre = log["indices"], log_o["indices"], log_o["pre_round"]
        bad = idx != idx_o
        near_tie = ((pre - pre.floor() - 0.5).abs() < 1e-4).any(dim=-1)
        far = int((bad & ~near_tie).sum())
        msg += f" FSQ ({len(levels)} levels) raw index mismatches {int(bad.sum())}/{bad.numel()}, {far} outside the tie band;"
        if far:
            fails.append(f"{far} FSQ index mismatches outside the 1e-4 tie band")
        if int(bad.sum()):
            # a code inside the tie band flipped: the other codes are checked, and the decoder on the codes the kernel chose
            zerr = zerr * (~bad)[:, None]
            with torch.no_grad():
                dec_o = om.decode(z.double())[:, :, -x.shape[2]:]
    else:
        kl, kl_o = float(log["kl_loss"]), float(log_o["kl_loss"])
        rel = abs(kl - kl_o) / abs(kl_o)
        msg += f" kl_loss rel err {rel:.2e} ({rel / 1e-4:.3f} of 1e-4);"
        if rel > 1e-4:
            fails.append(f"kl_loss {kl} vs {kl_o}")
    dz, dd = float(zerr.max()), float((dec.double() - dec_o).abs().max())
    msg += f" max|dz| {dz:.2e} max|ddec| {dd:.2e} (worst error / bound {max(dz, dd) / TOL:.3f})"
    if dz > TOL or dd > TOL:
        fails.append(f"exact: max|dz| {dz:.2e}, max|ddec| {dd:.2e} > {TOL}")
    del z, dec, log, zerr, dec_o, om

    # BF16 mode: PSNR against the input within the gate of the oracle's, and elementwise at bf16 noise level
    t0 = time.time()
    model.precision = "bf16"
    with torch.no_grad():
        torch.manual_seed(NOISE_SEED)
        _, dec, _ = model(xd)
    torch.cuda.synchronize()
    t_bf16 = time.time() - t0
    dec, ref = dec.cpu(), dec_oracle.float().cpu()
    p_new, p_ref = psnr01(x, dec), psnr01(x, ref)
    gate = 0.05 if fsq else 0.01
    dmax, dmean = float((dec - ref).abs().max()), float((dec - ref).abs().mean())
    ratio = abs(p_new - p_ref) / gate
    if not fsq:
        ratio = max(ratio, dmax / 0.25, dmean / 0.02)
    print(msg)
    print(f"[{case_id(case)}] bf16: PSNR {p_new:.4f} dB vs oracle {p_ref:.4f} dB; max|ddec| {dmax:.3f} mean|ddec| {dmean:.4f} "
          f"(worst error / bound {ratio:.3f})")
    print(f"[{case_id(case)}] wall: fp64 oracle {t_oracle:.1f} s, exact {t_exact:.1f} s, bf16 {t_bf16:.1f} s")
    if abs(p_new - p_ref) > gate:
        fails.append(f"bf16: PSNR {p_new:.4f} vs {p_ref:.4f}")
    if not fsq and (dmax > 0.25 or dmean > 0.02):
        fails.append(f"bf16: max|ddec| {dmax:.3f}, mean {dmean:.4f}")
    assert not fails, "\n".join(fails)


# ---------------------------------------------------------------------------------------------------------------
# plan keys of the zoo beyond PLAN_TABLE (one bf16 and one exact forward of every MODEL_CASES entry, B = 1, on an H100;
# test_zoo_forward_keys_are_in_tables lists any key missing here and any that no forward launches any more)
# ---------------------------------------------------------------------------------------------------------------
ZOO_PLAN_TABLE = [
    'conv_stem k333 3->128 @16x256x256 pad1.1',
    'conv_stem k333 3->128 @18x256x256',
    'conv_stem k333 3->128 @24x256x256',
    'conv_stem k333 3->128 @2x256x256',
    'conv_stem k333 3->128 @8x256x256',
    'conv_stem3 k333 3->128 @16x256x256 pad1.1',
    'conv_stem3 k333 3->128 @18x256x256',
    'conv_stem3 k333 3->128 @24x256x256',
    'conv_stem3 k333 3->128 @2x256x256',
    'conv_stem3 k333 3->128 @8x256x256',
    'conv_tc k111 s11 128->128 @16x256x256 tile1x8x16 bn128 ln0 r0 p1 t0 st6',
    'conv_tc k111 s11 128->128 @18x256x256 tile1x8x16 bn128 ln0 r0 p1 t0 st6',
    'conv_tc k111 s11 128->256 @12x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k111 s11 128->256 @18x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k111 s11 128->256 @2x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k111 s11 128->256 @8x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k111 s11 256->128 @18x256x256 tile1x8x16 bn128 ln0 r0 p1 t0 st6',
    'conv_tc k111 s11 256->128 @24x256x256 tile1x8x16 bn128 ln0 r0 p1 t0 st6',
    'conv_tc k111 s11 256->128 @4x256x256 tile1x8x16 bn128 ln0 r0 p1 t0 st6',
    'conv_tc k111 s11 256->512 @10x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k111 s11 256->512 @16x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k111 s11 256->512 @1x16x16 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k111 s11 256->512 @1x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k111 s11 256->512 @20x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k111 s11 256->512 @4x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k111 s11 256->512 @6x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k111 s11 256->512 @9x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k111 s11 512->256 @12x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k111 s11 512->256 @16x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k111 s11 512->256 @18x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k111 s11 512->256 @1x16x16 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k111 s11 512->512 @1x16x16 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k111 s11 512->512 @1x16x16 tile1x8x16 bn256 ln0 r1m p1 t0 st4',
    'conv_tc k111 s11 512->512 @2x16x16 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k111 s11 512->512 @2x16x16 tile1x8x16 bn256 ln0 r1m p1 t0 st4',
    'conv_tc k111 s11 512->512 @3x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k111 s11 512->512 @3x32x32 tile1x8x16 bn256 ln0 r1m p1 t0 st4',
    'conv_tc k111 s11 512->512 @4x16x16 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k111 s11 512->512 @4x16x16 tile1x8x16 bn256 ln0 r1m p1 t0 st4',
    'conv_tc k111 s11 512->512 @5x16x16 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k111 s11 512->512 @5x16x16 tile1x8x16 bn256 ln0 r1m p1 t0 st4',
    'conv_tc k111 s11 512->512 @5x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k111 s11 512->512 @5x64x64 tile1x8x16 bn256 ln0 r1m p1 t0 st4',
    'conv_tc k111 s11 512->512 @8x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k111 s11 512->512 @8x32x32 tile1x8x16 bn256 ln0 r1m p1 t0 st4',
    'conv_tc k111 s11 512->512 @9x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k111 s11 512->512 @9x32x32 tile1x8x16 bn256 ln0 r1m p1 t0 st4',
    'conv_tc k122 s11 256->256 @12x128x128 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k122 s11 256->256 @16x128x128 tile1x16x8 bn256 halo ln2 r0 p1 t0 st4',
    'conv_tc k122 s11 256->256 @18x128x128 tile1x16x8 bn256 halo ln2 r0 p1 t0 st4',
    'conv_tc k122 s11 256->256 @4x128x128 tile1x16x8 bn256 halo ln2 r0 p1 t0 st4',
    'conv_tc k122 s11 512->512 @2x16x16 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k122 s11 512->512 @3x32x32 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k122 s11 512->512 @4x16x16 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k122 s11 512->512 @5x16x16 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k122 s11 512->512 @6x64x64 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k122 s11 512->512 @8x32x32 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k122 s11 512->512 @8x64x64 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k122 s11 512->512 @9x32x32 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k122 s11 512->512 @9x64x64 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k133 s11 128->128 @18x256x256 tile1x16x8 bn128 halo ln1 r0 p1 t0 st8',
    'conv_tc k133 s11 128->128 @18x256x256 tile1x16x8 bn128 halo ln2 r1m p1 t0 st8',
    'conv_tc k133 s11 128->128 @24x256x256 tile1x16x8 bn128 halo ln1 r0 p1 t0 st8',
    'conv_tc k133 s11 128->128 @24x256x256 tile1x16x8 bn128 halo ln2 r1m p1 t0 st8',
    'conv_tc k133 s11 128->128 @2x256x256 tile1x16x8 bn128 halo ln1 r0 p1 t0 st8',
    'conv_tc k133 s11 128->128 @2x256x256 tile1x16x8 bn128 halo ln2 r1m p1 t0 st8',
    'conv_tc k133 s11 128->256 @12x128x128 tile1x16x8 bn256 halo ln1 r0 p1 t0 st4',
    'conv_tc k133 s11 128->256 @18x128x128 tile1x16x8 bn256 halo ln1 r0 p1 t0 st4',
    'conv_tc k133 s11 128->256 @2x128x128 tile1x16x8 bn256 halo ln1 r0 p1 t0 st4',
    'conv_tc k133 s11 128->256 @8x128x128 tile1x16x8 bn256 halo ln1 r0 p1 t0 st4',
    'conv_tc k133 s11 256->128 @18x256x256 tile1x16x8 bn128 halo ln1 r0 p1 t0 st8',
    'conv_tc k133 s11 256->128 @24x256x256 tile1x16x8 bn128 halo ln1 r0 p1 t0 st8',
    'conv_tc k133 s11 256->128 @4x256x256 tile1x16x8 bn128 halo ln1 r0 p1 t0 st8',
    'conv_tc k133 s11 256->256 @12x128x128 tile1x16x8 bn256 halo ln1 r0 p1 t0 st4',
    'conv_tc k133 s11 256->256 @12x128x128 tile1x16x8 bn256 halo ln2 r1m p1 t0 st4',
    'conv_tc k133 s11 256->256 @18x128x128 tile1x16x8 bn256 halo ln1 r0 p1 t0 st4',
    'conv_tc k133 s11 256->256 @18x128x128 tile1x16x8 bn256 halo ln2 r1m p1 t0 st4',
    'conv_tc k133 s11 256->256 @2x128x128 tile1x16x8 bn256 halo ln1 r0 p1 t0 st4',
    'conv_tc k133 s11 256->256 @2x128x128 tile1x16x8 bn256 halo ln2 r1m p1 t0 st4',
    'conv_tc k133 s11 256->512 @10x128x128 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k133 s11 256->512 @16x64x64 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k133 s11 256->512 @1x64x64 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k133 s11 256->512 @20x64x64 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k133 s11 256->512 @4x64x64 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k133 s11 256->512 @6x64x64 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k133 s11 256->512 @9x64x64 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k133 s11 512->256 @12x128x128 tile1x16x8 bn256 halo ln1 r0 p1 t0 st4',
    'conv_tc k133 s11 512->256 @16x128x128 tile1x16x8 bn256 halo ln1 r0 p1 t0 st4',
    'conv_tc k133 s11 512->256 @18x128x128 tile1x16x8 bn256 halo ln1 r0 p1 t0 st4',
    'conv_tc k133 s11 512->512 @10x128x128 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k133 s11 512->512 @10x128x128 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4',
    'conv_tc k133 s11 512->512 @10x32x32 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k133 s11 512->512 @10x32x32 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4',
    'conv_tc k133 s11 512->512 @16x64x64 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k133 s11 512->512 @16x64x64 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4',
    'conv_tc k133 s11 512->512 @1x16x16 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k133 s11 512->512 @1x16x16 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4',
    'conv_tc k133 s11 512->512 @1x64x64 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k133 s11 512->512 @1x64x64 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4',
    'conv_tc k133 s11 512->512 @20x64x64 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k133 s11 512->512 @20x64x64 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4',
    'conv_tc k133 s11 512->512 @2x16x16 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k133 s11 512->512 @2x16x16 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4',
    'conv_tc k133 s11 512->512 @3x32x32 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k133 s11 512->512 @3x32x32 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4',
    'conv_tc k133 s11 512->512 @4x16x16 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k133 s11 512->512 @4x16x16 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4',
    'conv_tc k133 s11 512->512 @5x16x16 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k133 s11 512->512 @5x16x16 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4',
    'conv_tc k133 s11 512->512 @6x64x64 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k133 s11 512->512 @6x64x64 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4',
    'conv_tc k133 s11 512->512 @8x32x32 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k133 s11 512->512 @8x32x32 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4',
    'conv_tc k133 s11 512->512 @9x32x32 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k133 s11 512->512 @9x32x32 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4',
    'conv_tc k133 s11 512->512 @9x64x64 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k133 s11 512->512 @9x64x64 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4',
    'conv_tc k133 s12 128->128 @16x128x128 tile1x8x16 bn128 ln0 r0 p1 t0 st6',
    'conv_tc k133 s12 128->128 @18x128x128 tile1x8x16 bn128 ln2 r0 p1 t0 st6',
    'conv_tc k133 s12 128->128 @24x128x128 tile1x8x16 bn128 ln0 r0 p1 t0 st6',
    'conv_tc k133 s12 128->128 @2x128x128 tile1x8x16 bn128 ln2 r0 p1 t0 st6',
    'conv_tc k133 s12 128->128 @8x128x128 tile1x8x16 bn128 ln0 r0 p1 t0 st6',
    'conv_tc k133 s12 256->256 @12x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k133 s12 256->256 @16x64x64 tile1x8x16 bn256 ln2 r0 p1 t0 st4',
    'conv_tc k133 s12 256->256 @18x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k133 s12 256->256 @20x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k133 s12 256->256 @20x64x64 tile1x8x16 bn256 ln2 r0 p1 t0 st4',
    'conv_tc k133 s12 256->256 @2x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k133 s12 256->256 @4x64x64 tile1x8x16 bn256 ln2 r0 p1 t0 st4',
    'conv_tc k133 s12 256->256 @8x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k133 s12 512->512 @10x16x16 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k133 s12 512->512 @10x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k133 s12 512->512 @16x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k133 s12 512->512 @1x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k133 s12 512->512 @20x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k133 s12 512->512 @2x16x16 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k133 s12 512->512 @4x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k133 s12 512->512 @6x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k133 s12 512->512 @8x16x16 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k133 s12 512->512 @9x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k233 s11 256->256 @8x256x256 tile1x16x8 bn256 halo ln2 r1 p1 t0 st4',
    'conv_tc k233 s11 256->256 @8x256x256 tile1x16x8 bn256 halo ln2 r1 p1 t0 st4 pad0.1',
    'conv_tc k233 s11 512->512 @4x128x128 tile1x16x8 bn256 halo ln0 r1 p1 t0 st4',
    'conv_tc k233 s11 512->512 @4x128x128 tile1x16x8 bn256 halo ln0 r1 p1 t0 st4 pad0.1',
    'conv_tc k233 s11 512->512 @9x128x128 tile1x16x8 bn256 halo ln0 r1 p1 t0 st4',
    'conv_tc k311 s11 128->128 @16x256x256 tile1x8x16 bn128 ln0 r1m p1 t0 st6 pad1.1',
    'conv_tc k311 s11 128->128 @16x256x256 tile1x8x16 bn128 ln1 r0 p1 t0 st6 pad1.1',
    'conv_tc k311 s11 128->128 @16x256x256 tile1x8x16 bn128 ln1 r0 p1 t1 st6',
    'conv_tc k311 s11 128->128 @16x256x256 tile1x8x16 bn128 ln2 r1m p1 t0 st6 pad1.1',
    'conv_tc k311 s11 128->128 @16x256x256 tile1x8x16 bn128 ln2 r1m p1 t1 st6',
    'conv_tc k311 s11 128->128 @18x256x256 tile1x8x16 bn128 ln0 r1m p1 t1 st6',
    'conv_tc k311 s11 128->128 @18x256x256 tile1x8x16 bn128 ln1 r0 p1 t1 st6',
    'conv_tc k311 s11 128->128 @18x256x256 tile1x8x16 bn128 ln1 r0 p1 t2 st6',
    'conv_tc k311 s11 128->128 @18x256x256 tile1x8x16 bn128 ln2 r1m p1 t1 st6',
    'conv_tc k311 s11 128->128 @18x256x256 tile1x8x16 bn128 ln2 r1m p1 t2 st6',
    'conv_tc k311 s11 128->128 @20x256x256 tile1x8x16 bn128 ln0 r1m p1 t1 st6',
    'conv_tc k311 s11 128->128 @20x256x256 tile1x8x16 bn128 ln1 r0 p1 t1 st6',
    'conv_tc k311 s11 128->128 @20x256x256 tile1x8x16 bn128 ln2 r1m p1 t1 st6',
    'conv_tc k311 s11 128->128 @24x256x256 tile1x8x16 bn128 ln0 r1m p1 t1 st6',
    'conv_tc k311 s11 128->128 @24x256x256 tile1x8x16 bn128 ln1 r0 p1 t1 st6',
    'conv_tc k311 s11 128->128 @24x256x256 tile1x8x16 bn128 ln1 r0 p1 t2 st6',
    'conv_tc k311 s11 128->128 @24x256x256 tile1x8x16 bn128 ln2 r1m p1 t1 st6',
    'conv_tc k311 s11 128->128 @24x256x256 tile1x8x16 bn128 ln2 r1m p1 t2 st6',
    'conv_tc k311 s11 128->128 @2x256x256 tile1x8x16 bn128 ln0 r1m p1 t1 st6',
    'conv_tc k311 s11 128->128 @2x256x256 tile1x8x16 bn128 ln1 r0 p1 t1 st6',
    'conv_tc k311 s11 128->128 @2x256x256 tile1x8x16 bn128 ln2 r1m p1 t1 st6',
    'conv_tc k311 s11 128->128 @8x256x256 tile1x8x16 bn128 ln0 r1m p1 t1 st6',
    'conv_tc k311 s11 256->256 @10x128x128 tile1x8x16 bn256 ln0 r1m p1 t1 st4',
    'conv_tc k311 s11 256->256 @10x128x128 tile1x8x16 bn256 ln1 r0 p1 t1 st4',
    'conv_tc k311 s11 256->256 @10x128x128 tile1x8x16 bn256 ln2 r1m p1 t1 st4',
    'conv_tc k311 s11 256->256 @12x128x128 tile1x8x16 bn256 ln0 r1m p1 t1 st4',
    'conv_tc k311 s11 256->256 @12x128x128 tile1x8x16 bn256 ln0 r1m p1 t2 st4',
    'conv_tc k311 s11 256->256 @12x128x128 tile1x8x16 bn256 ln1 r0 p1 t1 st4',
    'conv_tc k311 s11 256->256 @12x128x128 tile1x8x16 bn256 ln1 r0 p1 t2 st4',
    'conv_tc k311 s11 256->256 @12x128x128 tile1x8x16 bn256 ln2 r1m p1 t1 st4',
    'conv_tc k311 s11 256->256 @12x128x128 tile1x8x16 bn256 ln2 r1m p1 t2 st4',
    'conv_tc k311 s11 256->256 @16x128x128 tile1x8x16 bn256 ln0 r1m p1 t0 st4 pad1.1',
    'conv_tc k311 s11 256->256 @16x128x128 tile1x8x16 bn256 ln1 r0 p1 t0 st4 pad1.1',
    'conv_tc k311 s11 256->256 @16x128x128 tile1x8x16 bn256 ln2 r1m p1 t0 st4 pad1.1',
    'conv_tc k311 s11 256->256 @18x128x128 tile1x8x16 bn256 ln0 r1m p1 t0 st4',
    'conv_tc k311 s11 256->256 @18x128x128 tile1x8x16 bn256 ln0 r1m p1 t1 st4',
    'conv_tc k311 s11 256->256 @18x128x128 tile1x8x16 bn256 ln0 r1m p1 t2 st4',
    'conv_tc k311 s11 256->256 @18x128x128 tile1x8x16 bn256 ln1 r0 p1 t0 st4',
    'conv_tc k311 s11 256->256 @18x128x128 tile1x8x16 bn256 ln1 r0 p1 t1 st4',
    'conv_tc k311 s11 256->256 @18x128x128 tile1x8x16 bn256 ln1 r0 p1 t2 st4',
    'conv_tc k311 s11 256->256 @18x128x128 tile1x8x16 bn256 ln2 r1m p1 t0 st4',
    'conv_tc k311 s11 256->256 @18x128x128 tile1x8x16 bn256 ln2 r1m p1 t1 st4',
    'conv_tc k311 s11 256->256 @18x128x128 tile1x8x16 bn256 ln2 r1m p1 t2 st4',
    'conv_tc k311 s11 256->256 @20x128x128 tile1x8x16 bn256 ln0 r1m p1 t1 st4',
    'conv_tc k311 s11 256->256 @20x128x128 tile1x8x16 bn256 ln1 r0 p1 t1 st4',
    'conv_tc k311 s11 256->256 @20x128x128 tile1x8x16 bn256 ln2 r1m p1 t1 st4',
    'conv_tc k311 s11 256->256 @2x128x128 tile1x8x16 bn256 ln0 r1m p1 t1 st4',
    'conv_tc k311 s11 256->256 @2x128x128 tile1x8x16 bn256 ln1 r0 p1 t1 st4',
    'conv_tc k311 s11 256->256 @2x128x128 tile1x8x16 bn256 ln2 r1m p1 t1 st4',
    'conv_tc k311 s11 256->256 @8x128x128 tile1x8x16 bn256 ln0 r1m p1 t0 st4 pad1.1',
    'conv_tc k311 s11 256->256 @8x128x128 tile1x8x16 bn256 ln0 r1m p1 t1 st4',
    'conv_tc k311 s11 256->256 @8x128x128 tile1x8x16 bn256 ln1 r0 p1 t0 st4 pad1.1',
    'conv_tc k311 s11 256->256 @8x128x128 tile1x8x16 bn256 ln1 r0 p1 t1 st4',
    'conv_tc k311 s11 256->256 @8x128x128 tile1x8x16 bn256 ln2 r1m p1 t0 st4 pad1.1',
    'conv_tc k311 s11 256->256 @8x128x128 tile1x8x16 bn256 ln2 r1m p1 t1 st4',
    'conv_tc k311 s11 512->512 @10x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k311 s11 512->512 @10x128x128 tile1x8x16 bn256 ln0 r1m p1 t0 st4',
    'conv_tc k311 s11 512->512 @10x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k311 s11 512->512 @10x32x32 tile1x8x16 bn256 ln0 r0 p1 t1 st4',
    'conv_tc k311 s11 512->512 @10x32x32 tile1x8x16 bn256 ln0 r1m p1 t0 st4',
    'conv_tc k311 s11 512->512 @10x32x32 tile1x8x16 bn256 ln0 r1m p1 t1 st4',
    'conv_tc k311 s11 512->512 @10x64x64 tile1x8x16 bn256 ln0 r0 p1 t1 st4',
    'conv_tc k311 s11 512->512 @10x64x64 tile1x8x16 bn256 ln0 r1m p1 t1 st4',
    'conv_tc k311 s11 512->512 @16x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st4 pad1.1',
    'conv_tc k311 s11 512->512 @16x64x64 tile1x8x16 bn256 ln0 r0 p1 t2 st4',
    'conv_tc k311 s11 512->512 @16x64x64 tile1x8x16 bn256 ln0 r1m p1 t0 st4 pad1.1',
    'conv_tc k311 s11 512->512 @16x64x64 tile1x8x16 bn256 ln0 r1m p1 t2 st4',
    'conv_tc k311 s11 512->512 @1x16x16 tile1x8x16 bn256 ln0 r0 p1 t1 st4',
    'conv_tc k311 s11 512->512 @1x16x16 tile1x8x16 bn256 ln0 r1m p1 t1 st4',
    'conv_tc k311 s11 512->512 @1x64x64 tile1x8x16 bn256 ln0 r0 p1 t1 st4',
    'conv_tc k311 s11 512->512 @1x64x64 tile1x8x16 bn256 ln0 r1m p1 t1 st4',
    'conv_tc k311 s11 512->512 @20x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k311 s11 512->512 @20x64x64 tile1x8x16 bn256 ln0 r0 p1 t1 st4',
    'conv_tc k311 s11 512->512 @20x64x64 tile1x8x16 bn256 ln0 r1m p1 t0 st4',
    'conv_tc k311 s11 512->512 @20x64x64 tile1x8x16 bn256 ln0 r1m p1 t1 st4',
    'conv_tc k311 s11 512->512 @2x16x16 tile1x8x16 bn256 ln0 r0 p1 t1 st4',
    'conv_tc k311 s11 512->512 @2x16x16 tile1x8x16 bn256 ln0 r1m p1 t1 st4',
    'conv_tc k311 s11 512->512 @2x32x32 tile1x8x16 bn256 ln0 r0 p1 t2 st4',
    'conv_tc k311 s11 512->512 @2x32x32 tile1x8x16 bn256 ln0 r1m p1 t2 st4',
    'conv_tc k311 s11 512->512 @3x32x32 tile1x8x16 bn256 ln0 r0 p1 t1 st4',
    'conv_tc k311 s11 512->512 @3x32x32 tile1x8x16 bn256 ln0 r0 p1 t2 st4',
    'conv_tc k311 s11 512->512 @3x32x32 tile1x8x16 bn256 ln0 r1m p1 t1 st4',
    'conv_tc k311 s11 512->512 @3x32x32 tile1x8x16 bn256 ln0 r1m p1 t2 st4',
    'conv_tc k311 s11 512->512 @4x16x16 tile1x8x16 bn256 ln0 r0 p1 t0 st4 pad1.1',
    'conv_tc k311 s11 512->512 @4x16x16 tile1x8x16 bn256 ln0 r0 p1 t2 st4',
    'conv_tc k311 s11 512->512 @4x16x16 tile1x8x16 bn256 ln0 r1m p1 t0 st4 pad1.1',
    'conv_tc k311 s11 512->512 @4x16x16 tile1x8x16 bn256 ln0 r1m p1 t2 st4',
    'conv_tc k311 s11 512->512 @4x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st4 pad1.1',
    'conv_tc k311 s11 512->512 @4x32x32 tile1x8x16 bn256 ln0 r1m p1 t0 st4 pad1.1',
    'conv_tc k311 s11 512->512 @4x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st4 pad1.1',
    'conv_tc k311 s11 512->512 @4x64x64 tile1x8x16 bn256 ln0 r0 p1 t1 st4',
    'conv_tc k311 s11 512->512 @4x64x64 tile1x8x16 bn256 ln0 r1m p1 t0 st4 pad1.1',
    'conv_tc k311 s11 512->512 @4x64x64 tile1x8x16 bn256 ln0 r1m p1 t1 st4',
    'conv_tc k311 s11 512->512 @5x16x16 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k311 s11 512->512 @5x16x16 tile1x8x16 bn256 ln0 r0 p1 t1 st4',
    'conv_tc k311 s11 512->512 @5x16x16 tile1x8x16 bn256 ln0 r0 p1 t2 st4',
    'conv_tc k311 s11 512->512 @5x16x16 tile1x8x16 bn256 ln0 r1m p1 t0 st4',
    'conv_tc k311 s11 512->512 @5x16x16 tile1x8x16 bn256 ln0 r1m p1 t1 st4',
    'conv_tc k311 s11 512->512 @5x16x16 tile1x8x16 bn256 ln0 r1m p1 t2 st4',
    'conv_tc k311 s11 512->512 @5x32x32 tile1x8x16 bn256 ln0 r0 p1 t1 st4',
    'conv_tc k311 s11 512->512 @5x32x32 tile1x8x16 bn256 ln0 r1m p1 t1 st4',
    'conv_tc k311 s11 512->512 @5x64x64 tile1x8x16 bn256 ln0 r0 p1 t1 st4',
    'conv_tc k311 s11 512->512 @5x64x64 tile1x8x16 bn256 ln0 r1m p1 t1 st4',
    'conv_tc k311 s11 512->512 @6x64x64 tile1x8x16 bn256 ln0 r0 p1 t1 st4',
    'conv_tc k311 s11 512->512 @6x64x64 tile1x8x16 bn256 ln0 r0 p1 t2 st4',
    'conv_tc k311 s11 512->512 @6x64x64 tile1x8x16 bn256 ln0 r1m p1 t1 st4',
    'conv_tc k311 s11 512->512 @6x64x64 tile1x8x16 bn256 ln0 r1m p1 t2 st4',
    'conv_tc k311 s11 512->512 @8x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st4 pad1.1',
    'conv_tc k311 s11 512->512 @8x32x32 tile1x8x16 bn256 ln0 r0 p1 t2 st4',
    'conv_tc k311 s11 512->512 @8x32x32 tile1x8x16 bn256 ln0 r1m p1 t0 st4 pad1.1',
    'conv_tc k311 s11 512->512 @8x32x32 tile1x8x16 bn256 ln0 r1m p1 t2 st4',
    'conv_tc k311 s11 512->512 @8x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st4 pad1.1',
    'conv_tc k311 s11 512->512 @8x64x64 tile1x8x16 bn256 ln0 r1m p1 t0 st4 pad1.1',
    'conv_tc k311 s11 512->512 @9x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k311 s11 512->512 @9x32x32 tile1x8x16 bn256 ln0 r0 p1 t1 st4',
    'conv_tc k311 s11 512->512 @9x32x32 tile1x8x16 bn256 ln0 r0 p1 t2 st4',
    'conv_tc k311 s11 512->512 @9x32x32 tile1x8x16 bn256 ln0 r1m p1 t0 st4',
    'conv_tc k311 s11 512->512 @9x32x32 tile1x8x16 bn256 ln0 r1m p1 t1 st4',
    'conv_tc k311 s11 512->512 @9x32x32 tile1x8x16 bn256 ln0 r1m p1 t2 st4',
    'conv_tc k311 s11 512->512 @9x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st4',
    'conv_tc k311 s11 512->512 @9x64x64 tile1x8x16 bn256 ln0 r0 p1 t1 st4',
    'conv_tc k311 s11 512->512 @9x64x64 tile1x8x16 bn256 ln0 r0 p1 t2 st4',
    'conv_tc k311 s11 512->512 @9x64x64 tile1x8x16 bn256 ln0 r1m p1 t0 st4',
    'conv_tc k311 s11 512->512 @9x64x64 tile1x8x16 bn256 ln0 r1m p1 t1 st4',
    'conv_tc k311 s11 512->512 @9x64x64 tile1x8x16 bn256 ln0 r1m p1 t2 st4',
    'conv_tc k333 s11 128->3 @16x256x256 tile1x16x8 bn32 halo ln0 r0 p1 t1 st8',
    'conv_tc k333 s11 128->3 @18x256x256 tile1x16x8 bn32 halo ln0 r0 p1 t1 st8',
    'conv_tc k333 s11 128->3 @18x256x256 tile1x16x8 bn32 halo ln0 r0 p1 t2 st8',
    'conv_tc k333 s11 128->3 @20x256x256 tile1x16x8 bn32 halo ln0 r0 p1 t1 st8',
    'conv_tc k333 s11 128->3 @24x256x256 tile1x16x8 bn32 halo ln0 r0 p1 t1 st8',
    'conv_tc k333 s11 128->3 @24x256x256 tile1x16x8 bn32 halo ln0 r0 p1 t2 st8',
    'conv_tc k333 s11 128->3 @4x256x256 tile1x16x8 bn32 halo ln0 r0 p1 t1 st8',
    'conv_tc k333 s11 256->256 @16x256x256 tile1x16x8 bn256 halo ln2 r1 p1 t1 st4',
    'conv_tc k333 s11 256->256 @20x256x256 tile1x16x8 bn256 halo ln2 r1 p1 t1 st4',
    'conv_tc k333 s11 256->256 @24x256x256 tile1x16x8 bn256 halo ln2 r1 p1 t1 st4',
    'conv_tc k333 s11 256->256 @24x256x256 tile1x16x8 bn256 halo ln2 r1 p1 t2 st4',
    'conv_tc k333 s11 512->16 @1x32x32 tile1x16x8 bn32 halo ln0 r0 p1 t1 st8',
    'conv_tc k333 s11 512->16 @5x32x32 tile1x16x8 bn32 halo ln0 r0 p1 t0 st8',
    'conv_tc k333 s11 512->16 @8x32x32 tile1x16x8 bn32 halo ln0 r0 p1 t2 st8',
    'conv_tc k333 s11 512->16 @9x32x32 tile1x16x8 bn32 halo ln0 r0 p1 t0 st8',
    'conv_tc k333 s11 512->16 @9x32x32 tile1x16x8 bn32 halo ln0 r0 p1 t1 st8',
    'conv_tc k333 s11 512->32 @1x16x16 tile1x16x8 bn32 halo ln0 r0 p1 t1 st8',
    'conv_tc k333 s11 512->32 @4x16x16 tile1x16x8 bn32 halo ln0 r0 p1 t0 st8 pad1.1',
    'conv_tc k333 s11 512->32 @4x16x16 tile1x16x8 bn32 halo ln0 r0 p1 t2 st8',
    'conv_tc k333 s11 512->32 @4x32x32 tile1x16x8 bn32 halo ln0 r0 p1 t0 st8 pad1.1',
    'conv_tc k333 s11 512->32 @5x16x16 tile1x16x8 bn32 halo ln0 r0 p1 t1 st8',
    'conv_tc k333 s11 512->32 @5x32x32 tile1x16x8 bn32 halo ln0 r0 p1 t0 st8',
    'conv_tc k333 s11 512->32 @5x32x32 tile1x16x8 bn32 halo ln0 r0 p1 t1 st8',
    'conv_tc k333 s11 512->4 @5x32x32 tile1x16x8 bn32 halo ln0 r0 p1 t0 st8',
    'conv_tc k333 s11 512->5 @1x32x32 tile1x16x8 bn32 halo ln0 r0 p1 t1 st8',
    'conv_tc k333 s11 512->5 @2x32x32 tile1x16x8 bn32 halo ln0 r0 p1 t2 st8',
    'conv_tc k333 s11 512->5 @3x32x32 tile1x16x8 bn32 halo ln0 r0 p1 t1 st8',
    'conv_tc k333 s11 512->5 @4x32x32 tile1x16x8 bn32 halo ln0 r0 p1 t2 st8',
    'conv_tc k333 s11 512->5 @5x32x32 tile1x16x8 bn32 halo ln0 r0 p1 t1 st8',
    'conv_tc k333 s11 512->512 @10x128x128 tile1x16x8 bn256 halo ln0 r1 p1 t1 st4',
    'conv_tc k333 s11 512->512 @12x128x128 tile1x16x8 bn256 halo ln0 r1 p1 t1 st4',
    'conv_tc k333 s11 512->512 @12x128x128 tile1x16x8 bn256 halo ln0 r1 p1 t2 st4',
    'conv_tc k333 s11 512->512 @16x128x128 tile1x16x8 bn256 halo ln0 r1 p1 t2 st4',
    'conv_tc k333 s11 512->512 @18x128x128 tile1x16x8 bn256 halo ln0 r1 p1 t1 st4',
    'conv_tc k333 s11 512->512 @18x128x128 tile1x16x8 bn256 halo ln0 r1 p1 t2 st4',
    'conv_tc k333 s11 512->512 @1x16x16 tile1x16x8 bn256 halo ln0 r0 p1 t1 st4',
    'conv_tc k333 s11 512->512 @1x16x16 tile1x16x8 bn256 halo ln0 r1m p1 t1 st4',
    'conv_tc k333 s11 512->512 @2x16x16 tile1x16x8 bn256 halo ln0 r0 p1 t1 st4',
    'conv_tc k333 s11 512->512 @2x16x16 tile1x16x8 bn256 halo ln0 r1m p1 t1 st4',
    'conv_tc k333 s11 512->512 @2x32x32 tile1x16x8 bn256 halo ln0 r0 p1 t2 st4',
    'conv_tc k333 s11 512->512 @2x32x32 tile1x16x8 bn256 halo ln0 r1m p1 t2 st4',
    'conv_tc k333 s11 512->512 @3x32x32 tile1x16x8 bn256 halo ln0 r0 p1 t1 st4',
    'conv_tc k333 s11 512->512 @3x32x32 tile1x16x8 bn256 halo ln0 r0 p1 t2 st4',
    'conv_tc k333 s11 512->512 @3x32x32 tile1x16x8 bn256 halo ln0 r1m p1 t1 st4',
    'conv_tc k333 s11 512->512 @3x32x32 tile1x16x8 bn256 halo ln0 r1m p1 t2 st4',
    'conv_tc k333 s11 512->512 @4x16x16 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4 pad1.1',
    'conv_tc k333 s11 512->512 @4x16x16 tile1x16x8 bn256 halo ln0 r0 p1 t2 st4',
    'conv_tc k333 s11 512->512 @4x16x16 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4 pad1.1',
    'conv_tc k333 s11 512->512 @4x16x16 tile1x16x8 bn256 halo ln0 r1m p1 t2 st4',
    'conv_tc k333 s11 512->512 @4x32x32 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4 pad1.1',
    'conv_tc k333 s11 512->512 @4x32x32 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4 pad1.1',
    'conv_tc k333 s11 512->512 @4x64x64 tile1x16x8 bn256 halo ln0 r1 p1 t1 st4',
    'conv_tc k333 s11 512->512 @4x64x64 tile1x16x8 bn256 halo ln0 r1 p1 t2 st4',
    'conv_tc k333 s11 512->512 @5x16x16 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k333 s11 512->512 @5x16x16 tile1x16x8 bn256 halo ln0 r0 p1 t1 st4',
    'conv_tc k333 s11 512->512 @5x16x16 tile1x16x8 bn256 halo ln0 r0 p1 t2 st4',
    'conv_tc k333 s11 512->512 @5x16x16 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4',
    'conv_tc k333 s11 512->512 @5x16x16 tile1x16x8 bn256 halo ln0 r1m p1 t1 st4',
    'conv_tc k333 s11 512->512 @5x16x16 tile1x16x8 bn256 halo ln0 r1m p1 t2 st4',
    'conv_tc k333 s11 512->512 @5x32x32 tile1x16x8 bn256 halo ln0 r0 p1 t1 st4',
    'conv_tc k333 s11 512->512 @5x32x32 tile1x16x8 bn256 halo ln0 r1m p1 t1 st4',
    'conv_tc k333 s11 512->512 @5x64x64 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k333 s11 512->512 @5x64x64 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4',
    'conv_tc k333 s11 512->512 @6x64x64 tile1x16x8 bn256 halo ln0 r1 p1 t1 st4',
    'conv_tc k333 s11 512->512 @6x64x64 tile1x16x8 bn256 halo ln0 r1 p1 t2 st4',
    'conv_tc k333 s11 512->512 @8x128x128 tile1x16x8 bn256 halo ln0 r1 p1 t1 st4',
    'conv_tc k333 s11 512->512 @8x32x32 tile1x16x8 bn256 halo ln0 r0 p1 t2 st4',
    'conv_tc k333 s11 512->512 @8x32x32 tile1x16x8 bn256 halo ln0 r1m p1 t2 st4',
    'conv_tc k333 s11 512->512 @9x32x32 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4',
    'conv_tc k333 s11 512->512 @9x32x32 tile1x16x8 bn256 halo ln0 r0 p1 t1 st4',
    'conv_tc k333 s11 512->512 @9x32x32 tile1x16x8 bn256 halo ln0 r0 p1 t2 st4',
    'conv_tc k333 s11 512->512 @9x32x32 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4',
    'conv_tc k333 s11 512->512 @9x32x32 tile1x16x8 bn256 halo ln0 r1m p1 t1 st4',
    'conv_tc k333 s11 512->512 @9x32x32 tile1x16x8 bn256 halo ln0 r1m p1 t2 st4',
    'conv_tc k333 s11 512->6 @1x16x16 tile1x16x8 bn32 halo ln0 r0 p1 t1 st8',
    'conv_tc k333 s11 512->6 @4x16x16 tile1x16x8 bn32 halo ln0 r0 p1 t0 st8 pad1.1',
    'conv_tc k333 s11 512->6 @4x16x16 tile1x16x8 bn32 halo ln0 r0 p1 t2 st8',
    'conv_tc k333 s11 512->6 @4x32x32 tile1x16x8 bn32 halo ln0 r0 p1 t0 st8 pad1.1',
    'conv_tc k333 s11 512->6 @5x16x16 tile1x16x8 bn32 halo ln0 r0 p1 t0 st8',
    'conv_tc k333 s11 512->6 @5x16x16 tile1x16x8 bn32 halo ln0 r0 p1 t1 st8',
    'conv_tc k333 s11 512->6 @5x32x32 tile1x16x8 bn32 halo ln0 r0 p1 t0 st8',
    'conv_tc k333 s11 512->8 @1x32x32 tile1x16x8 bn32 halo ln0 r0 p1 t1 st8',
    'conv_tc k333 s11 512->8 @4x16x16 tile1x16x8 bn32 halo ln0 r0 p1 t0 st8 pad1.1',
    'conv_tc k333 s11 512->8 @4x32x32 tile1x16x8 bn32 halo ln0 r0 p1 t0 st8 pad1.1',
    'conv_tc k333 s11 512->8 @4x32x32 tile1x16x8 bn32 halo ln0 r0 p1 t2 st8',
    'conv_tc k333 s11 512->8 @5x16x16 tile1x16x8 bn32 halo ln0 r0 p1 t0 st8',
    'conv_tc k333 s11 512->8 @5x32x32 tile1x16x8 bn32 halo ln0 r0 p1 t1 st8',
    'conv_tc k333 s11 512->8 @5x64x64 tile1x16x8 bn32 halo ln0 r0 p1 t0 st8',
    'conv_tc k333 s21 128->128 @12x128x128 tile1x16x8 bn128 halo ln2 r3 p1 t1 st8',
    'conv_tc k333 s21 128->128 @4x128x128 tile1x16x8 bn128 halo ln2 r3 p1 t1 st8',
    'conv_tc k333 s21 128->128 @8x128x128 tile1x16x8 bn128 halo ln2 r3 p1 t2 st8',
    'conv_tc k333 s21 256->256 @10x128x128 tile1x16x8 bn256 halo ln2 r3 p1 t0 st4',
    'conv_tc k333 s21 256->256 @10x64x64 tile1x16x8 bn256 halo ln2 r3 p1 t1 st4',
    'conv_tc k333 s21 256->256 @1x64x64 tile1x16x8 bn256 halo ln2 r3 p1 t1 st4',
    'conv_tc k333 s21 256->256 @4x64x64 tile1x16x8 bn256 halo ln2 r3 p1 t2 st4',
    'conv_tc k333 s21 256->256 @6x64x64 tile1x16x8 bn256 halo ln2 r3 p1 t1 st4',
    'conv_tc k333 s21 256->256 @8x64x64 tile1x16x8 bn256 halo ln2 r3 p1 t0 st4 pad0.1 pool1',
    'conv_tc k333 s21 256->256 @9x64x64 tile1x16x8 bn256 halo ln2 r3 p1 t0 st4',
    'conv_tc k333 s21 256->256 @9x64x64 tile1x16x8 bn256 halo ln2 r3 p1 t1 st4',
    'conv_tc k333 s21 512->512 @10x32x32 tile1x16x8 bn256 halo ln0 r3 p1 t0 st4',
    'conv_tc k333 s21 512->512 @10x32x32 tile1x16x8 bn256 halo ln0 r3 p1 t1 st4',
    'conv_tc k333 s21 512->512 @1x16x16 tile1x16x8 bn256 halo ln0 r3 p1 t1 st4',
    'conv_tc k333 s21 512->512 @2x32x32 tile1x16x8 bn256 halo ln0 r3 p1 t1 st4',
    'conv_tc k333 s21 512->512 @2x32x32 tile1x16x8 bn256 halo ln0 r3 p1 t2 st4',
    'conv_tc k333 s21 512->512 @3x32x32 tile1x16x8 bn256 halo ln0 r3 p1 t1 st4',
    'conv_tc k333 s21 512->512 @4x16x16 tile1x16x8 bn256 halo ln0 r3 p1 t0 st4 pad0.1 pool1',
    'conv_tc k333 s21 512->512 @4x16x16 tile1x16x8 bn256 halo ln0 r3 p1 t2 st4',
    'conv_tc k333 s21 512->512 @4x32x32 tile1x16x8 bn256 halo ln0 r3 p1 t0 st4 pad0.1 pool1',
    'conv_tc k333 s21 512->512 @5x16x16 tile1x16x8 bn256 halo ln0 r3 p1 t0 st4',
    'conv_tc k333 s21 512->512 @5x16x16 tile1x16x8 bn256 halo ln0 r3 p1 t1 st4',
    'conv_tc k333 s21 512->512 @5x32x32 tile1x16x8 bn256 halo ln0 r3 p1 t1 st4',
    'conv_tc k333 s21 512->512 @5x64x64 tile1x16x8 bn256 halo ln0 r3 p1 t0 st4',
    'conv_tc k333 s21 512->512 @8x32x32 tile1x16x8 bn256 halo ln0 r3 p1 t0 st4 pad0.1 pool1',
    'conv_tc k333 s21 512->512 @8x32x32 tile1x16x8 bn256 halo ln0 r3 p1 t2 st4',
    'conv_tc3 k111 s11 128->256 @12x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st2',
    'conv_tc3 k111 s11 128->256 @18x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st2',
    'conv_tc3 k111 s11 128->256 @2x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st2',
    'conv_tc3 k111 s11 128->256 @8x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st2',
    'conv_tc3 k111 s11 256->128 @18x256x256 tile1x8x16 bn128 ln0 r0 p1 t0 st3',
    'conv_tc3 k111 s11 256->128 @24x256x256 tile1x8x16 bn128 ln0 r0 p1 t0 st3',
    'conv_tc3 k111 s11 256->128 @4x256x256 tile1x8x16 bn128 ln0 r0 p1 t0 st3',
    'conv_tc3 k111 s11 256->512 @10x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st2',
    'conv_tc3 k111 s11 256->512 @16x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st2',
    'conv_tc3 k111 s11 256->512 @1x16x16 tile1x8x16 bn256 ln0 r0 p1 t0 st2',
    'conv_tc3 k111 s11 256->512 @1x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st2',
    'conv_tc3 k111 s11 256->512 @20x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st2',
    'conv_tc3 k111 s11 256->512 @4x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st2',
    'conv_tc3 k111 s11 256->512 @6x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st2',
    'conv_tc3 k111 s11 256->512 @9x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st2',
    'conv_tc3 k111 s11 512->256 @12x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st2',
    'conv_tc3 k111 s11 512->256 @16x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st2',
    'conv_tc3 k111 s11 512->256 @18x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st2',
    'conv_tc3 k111 s11 512->256 @1x16x16 tile1x8x16 bn256 ln0 r0 p1 t0 st2',
    'conv_tc3 k111 s11 512->512 @1x16x16 tile1x8x16 bn256 ln0 r0 p1 t0 st2',
    'conv_tc3 k111 s11 512->512 @1x16x16 tile1x8x16 bn256 ln0 r1m p1 t0 st2',
    'conv_tc3 k111 s11 512->512 @2x16x16 tile1x8x16 bn256 ln0 r0 p1 t0 st2',
    'conv_tc3 k111 s11 512->512 @2x16x16 tile1x8x16 bn256 ln0 r1m p1 t0 st2',
    'conv_tc3 k111 s11 512->512 @3x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st2',
    'conv_tc3 k111 s11 512->512 @3x32x32 tile1x8x16 bn256 ln0 r1m p1 t0 st2',
    'conv_tc3 k111 s11 512->512 @4x16x16 tile1x8x16 bn256 ln0 r0 p1 t0 st2',
    'conv_tc3 k111 s11 512->512 @4x16x16 tile1x8x16 bn256 ln0 r1m p1 t0 st2',
    'conv_tc3 k111 s11 512->512 @5x16x16 tile1x8x16 bn256 ln0 r0 p1 t0 st2',
    'conv_tc3 k111 s11 512->512 @5x16x16 tile1x8x16 bn256 ln0 r1m p1 t0 st2',
    'conv_tc3 k111 s11 512->512 @5x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st2',
    'conv_tc3 k111 s11 512->512 @5x64x64 tile1x8x16 bn256 ln0 r1m p1 t0 st2',
    'conv_tc3 k111 s11 512->512 @8x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st2',
    'conv_tc3 k111 s11 512->512 @8x32x32 tile1x8x16 bn256 ln0 r1m p1 t0 st2',
    'conv_tc3 k111 s11 512->512 @9x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st2',
    'conv_tc3 k111 s11 512->512 @9x32x32 tile1x8x16 bn256 ln0 r1m p1 t0 st2',
    'conv_tc3 k122 s11 256->256 @12x128x128 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2',
    'conv_tc3 k122 s11 256->256 @16x128x128 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2',
    'conv_tc3 k122 s11 256->256 @18x128x128 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2',
    'conv_tc3 k122 s11 512->512 @2x16x16 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2',
    'conv_tc3 k122 s11 512->512 @3x32x32 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2',
    'conv_tc3 k122 s11 512->512 @4x16x16 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2',
    'conv_tc3 k122 s11 512->512 @5x16x16 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2',
    'conv_tc3 k122 s11 512->512 @6x64x64 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2',
    'conv_tc3 k122 s11 512->512 @8x32x32 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2',
    'conv_tc3 k122 s11 512->512 @8x64x64 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2',
    'conv_tc3 k122 s11 512->512 @9x32x32 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2',
    'conv_tc3 k122 s11 512->512 @9x64x64 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2',
    'conv_tc3 k133 s11 128->128 @18x256x256 tile1x16x8 bn128 halo ln1 r0 p4 t0 st2',
    'conv_tc3 k133 s11 128->128 @18x256x256 tile1x16x8 bn128 halo ln2 r1m p4 t0 st2',
    'conv_tc3 k133 s11 128->128 @24x256x256 tile1x16x8 bn128 halo ln1 r0 p4 t0 st2',
    'conv_tc3 k133 s11 128->128 @24x256x256 tile1x16x8 bn128 halo ln2 r1m p4 t0 st2',
    'conv_tc3 k133 s11 128->128 @2x256x256 tile1x16x8 bn128 halo ln1 r0 p4 t0 st2',
    'conv_tc3 k133 s11 128->128 @2x256x256 tile1x16x8 bn128 halo ln2 r1m p4 t0 st2',
    'conv_tc3 k133 s11 128->256 @12x128x128 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2',
    'conv_tc3 k133 s11 128->256 @18x128x128 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2',
    'conv_tc3 k133 s11 128->256 @2x128x128 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2',
    'conv_tc3 k133 s11 128->256 @8x128x128 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2',
    'conv_tc3 k133 s11 256->128 @18x256x256 tile1x16x8 bn128 halo ln1 r0 p4 t0 st2',
    'conv_tc3 k133 s11 256->128 @24x256x256 tile1x16x8 bn128 halo ln1 r0 p4 t0 st2',
    'conv_tc3 k133 s11 256->128 @4x256x256 tile1x16x8 bn128 halo ln1 r0 p4 t0 st2',
    'conv_tc3 k133 s11 256->256 @12x128x128 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2',
    'conv_tc3 k133 s11 256->256 @12x128x128 tile1x16x8 bn128 halo ln0 r1m p4 t0 st2',
    'conv_tc3 k133 s11 256->256 @18x128x128 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2',
    'conv_tc3 k133 s11 256->256 @18x128x128 tile1x16x8 bn128 halo ln0 r1m p4 t0 st2',
    'conv_tc3 k133 s11 256->256 @2x128x128 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2',
    'conv_tc3 k133 s11 256->256 @2x128x128 tile1x16x8 bn128 halo ln0 r1m p4 t0 st2',
    'conv_tc3 k133 s11 256->512 @10x128x128 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2',
    'conv_tc3 k133 s11 256->512 @16x64x64 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2',
    'conv_tc3 k133 s11 256->512 @1x64x64 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2',
    'conv_tc3 k133 s11 256->512 @20x64x64 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2',
    'conv_tc3 k133 s11 256->512 @4x64x64 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2',
    'conv_tc3 k133 s11 256->512 @6x64x64 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2',
    'conv_tc3 k133 s11 256->512 @9x64x64 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2',
    'conv_tc3 k133 s11 512->256 @12x128x128 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2',
    'conv_tc3 k133 s11 512->256 @16x128x128 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2',
    'conv_tc3 k133 s11 512->256 @18x128x128 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2',
    'conv_tc3 k133 s11 512->512 @10x128x128 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2',
    'conv_tc3 k133 s11 512->512 @10x128x128 tile1x16x8 bn128 halo ln0 r1m p8 t0 st2',
    'conv_tc3 k133 s11 512->512 @10x32x32 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2',
    'conv_tc3 k133 s11 512->512 @10x32x32 tile1x16x8 bn128 halo ln0 r1m p8 t0 st2',
    'conv_tc3 k133 s11 512->512 @16x64x64 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2',
    'conv_tc3 k133 s11 512->512 @16x64x64 tile1x16x8 bn128 halo ln0 r1m p8 t0 st2',
    'conv_tc3 k133 s11 512->512 @1x16x16 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2',
    'conv_tc3 k133 s11 512->512 @1x16x16 tile1x16x8 bn128 halo ln0 r1m p8 t0 st2',
    'conv_tc3 k133 s11 512->512 @1x64x64 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2',
    'conv_tc3 k133 s11 512->512 @1x64x64 tile1x16x8 bn128 halo ln0 r1m p8 t0 st2',
    'conv_tc3 k133 s11 512->512 @20x64x64 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2',
    'conv_tc3 k133 s11 512->512 @20x64x64 tile1x16x8 bn128 halo ln0 r1m p8 t0 st2',
    'conv_tc3 k133 s11 512->512 @2x16x16 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2',
    'conv_tc3 k133 s11 512->512 @2x16x16 tile1x16x8 bn128 halo ln0 r1m p8 t0 st2',
    'conv_tc3 k133 s11 512->512 @3x32x32 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2',
    'conv_tc3 k133 s11 512->512 @3x32x32 tile1x16x8 bn128 halo ln0 r1m p8 t0 st2',
    'conv_tc3 k133 s11 512->512 @4x16x16 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2',
    'conv_tc3 k133 s11 512->512 @4x16x16 tile1x16x8 bn128 halo ln0 r1m p8 t0 st2',
    'conv_tc3 k133 s11 512->512 @5x16x16 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2',
    'conv_tc3 k133 s11 512->512 @5x16x16 tile1x16x8 bn128 halo ln0 r1m p8 t0 st2',
    'conv_tc3 k133 s11 512->512 @6x64x64 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2',
    'conv_tc3 k133 s11 512->512 @6x64x64 tile1x16x8 bn128 halo ln0 r1m p8 t0 st2',
    'conv_tc3 k133 s11 512->512 @8x32x32 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2',
    'conv_tc3 k133 s11 512->512 @8x32x32 tile1x16x8 bn128 halo ln0 r1m p8 t0 st2',
    'conv_tc3 k133 s11 512->512 @9x32x32 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2',
    'conv_tc3 k133 s11 512->512 @9x32x32 tile1x16x8 bn128 halo ln0 r1m p8 t0 st2',
    'conv_tc3 k133 s11 512->512 @9x64x64 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2',
    'conv_tc3 k133 s11 512->512 @9x64x64 tile1x16x8 bn128 halo ln0 r1m p8 t0 st2',
    'conv_tc3 k133 s12 128->128 @16x128x128 tile1x8x16 bn128 ln0 r0 p4 t0 st3',
    'conv_tc3 k133 s12 128->128 @18x128x128 tile1x8x16 bn128 ln2 r0 p4 t0 st3',
    'conv_tc3 k133 s12 128->128 @24x128x128 tile1x8x16 bn128 ln0 r0 p4 t0 st3',
    'conv_tc3 k133 s12 128->128 @2x128x128 tile1x8x16 bn128 ln2 r0 p4 t0 st3',
    'conv_tc3 k133 s12 128->128 @8x128x128 tile1x8x16 bn128 ln0 r0 p4 t0 st3',
    'conv_tc3 k133 s12 256->256 @12x64x64 tile1x8x16 bn128 ln0 r0 p4 t0 st3',
    'conv_tc3 k133 s12 256->256 @18x64x64 tile1x8x16 bn128 ln0 r0 p4 t0 st3',
    'conv_tc3 k133 s12 256->256 @2x64x64 tile1x8x16 bn128 ln0 r0 p4 t0 st3',
    'conv_tc3 k133 s12 256->256 @8x64x64 tile1x8x16 bn128 ln0 r0 p4 t0 st3',
    'conv_tc3 k133 s12 512->512 @10x16x16 tile1x8x16 bn128 ln0 r0 p8 t0 st3',
    'conv_tc3 k133 s12 512->512 @10x64x64 tile1x8x16 bn128 ln0 r0 p8 t0 st3',
    'conv_tc3 k133 s12 512->512 @16x32x32 tile1x8x16 bn128 ln0 r0 p8 t0 st3',
    'conv_tc3 k133 s12 512->512 @1x32x32 tile1x8x16 bn128 ln0 r0 p8 t0 st3',
    'conv_tc3 k133 s12 512->512 @20x32x32 tile1x8x16 bn128 ln0 r0 p8 t0 st3',
    'conv_tc3 k133 s12 512->512 @2x16x16 tile1x8x16 bn128 ln0 r0 p8 t0 st3',
    'conv_tc3 k133 s12 512->512 @4x32x32 tile1x8x16 bn128 ln0 r0 p8 t0 st3',
    'conv_tc3 k133 s12 512->512 @6x32x32 tile1x8x16 bn128 ln0 r0 p8 t0 st3',
    'conv_tc3 k133 s12 512->512 @8x16x16 tile1x8x16 bn128 ln0 r0 p8 t0 st3',
    'conv_tc3 k133 s12 512->512 @9x32x32 tile1x8x16 bn128 ln0 r0 p8 t0 st3',
    'conv_tc3 k233 s11 256->256 @8x256x256 tile1x16x8 bn128 halo ln0 r1 p8 t0 st2',
    'conv_tc3 k233 s11 256->256 @8x256x256 tile1x16x8 bn128 halo ln0 r1 p8 t0 st2 pad0.1',
    'conv_tc3 k233 s11 512->512 @4x128x128 tile1x16x8 bn64 halo ln0 r1 p8 t0 st4',
    'conv_tc3 k233 s11 512->512 @4x128x128 tile1x16x8 bn64 halo ln0 r1 p8 t0 st4 pad0.1',
    'conv_tc3 k233 s11 512->512 @9x128x128 tile1x16x8 bn64 halo ln0 r1 p8 t0 st4',
    'conv_tc3 k311 s11 128->128 @16x256x256 tile1x8x16 bn128 ln0 r1m p1 t0 st3 pad1.1',
    'conv_tc3 k311 s11 128->128 @16x256x256 tile1x8x16 bn128 ln1 r0 p1 t0 st3 pad1.1',
    'conv_tc3 k311 s11 128->128 @16x256x256 tile1x8x16 bn128 ln1 r0 p1 t1 st3',
    'conv_tc3 k311 s11 128->128 @16x256x256 tile1x8x16 bn128 ln2 r1m p1 t0 st3 pad1.1',
    'conv_tc3 k311 s11 128->128 @16x256x256 tile1x8x16 bn128 ln2 r1m p1 t1 st3',
    'conv_tc3 k311 s11 128->128 @18x256x256 tile1x8x16 bn128 ln0 r1m p1 t0 st3',
    'conv_tc3 k311 s11 128->128 @18x256x256 tile1x8x16 bn128 ln0 r1m p1 t1 st3',
    'conv_tc3 k311 s11 128->128 @18x256x256 tile1x8x16 bn128 ln1 r0 p1 t0 st3',
    'conv_tc3 k311 s11 128->128 @18x256x256 tile1x8x16 bn128 ln1 r0 p1 t1 st3',
    'conv_tc3 k311 s11 128->128 @18x256x256 tile1x8x16 bn128 ln1 r0 p1 t2 st3',
    'conv_tc3 k311 s11 128->128 @18x256x256 tile1x8x16 bn128 ln2 r1m p1 t0 st3',
    'conv_tc3 k311 s11 128->128 @18x256x256 tile1x8x16 bn128 ln2 r1m p1 t1 st3',
    'conv_tc3 k311 s11 128->128 @18x256x256 tile1x8x16 bn128 ln2 r1m p1 t2 st3',
    'conv_tc3 k311 s11 128->128 @20x256x256 tile1x8x16 bn128 ln0 r1m p1 t1 st3',
    'conv_tc3 k311 s11 128->128 @20x256x256 tile1x8x16 bn128 ln1 r0 p1 t1 st3',
    'conv_tc3 k311 s11 128->128 @20x256x256 tile1x8x16 bn128 ln2 r1m p1 t1 st3',
    'conv_tc3 k311 s11 128->128 @24x256x256 tile1x8x16 bn128 ln0 r1m p1 t1 st3',
    'conv_tc3 k311 s11 128->128 @24x256x256 tile1x8x16 bn128 ln1 r0 p1 t1 st3',
    'conv_tc3 k311 s11 128->128 @24x256x256 tile1x8x16 bn128 ln1 r0 p1 t2 st3',
    'conv_tc3 k311 s11 128->128 @24x256x256 tile1x8x16 bn128 ln2 r1m p1 t1 st3',
    'conv_tc3 k311 s11 128->128 @24x256x256 tile1x8x16 bn128 ln2 r1m p1 t2 st3',
    'conv_tc3 k311 s11 128->128 @2x256x256 tile1x8x16 bn128 ln0 r1m p1 t1 st3',
    'conv_tc3 k311 s11 128->128 @2x256x256 tile1x8x16 bn128 ln1 r0 p1 t1 st3',
    'conv_tc3 k311 s11 128->128 @2x256x256 tile1x8x16 bn128 ln2 r1m p1 t1 st3',
    'conv_tc3 k311 s11 128->128 @8x256x256 tile1x8x16 bn128 ln0 r1m p1 t1 st3',
    'conv_tc3 k311 s11 256->256 @10x128x128 tile1x8x16 bn256 ln0 r1m p1 t1 st2',
    'conv_tc3 k311 s11 256->256 @10x128x128 tile1x8x16 bn256 ln1 r0 p1 t1 st2',
    'conv_tc3 k311 s11 256->256 @10x128x128 tile1x8x16 bn256 ln2 r1m p1 t1 st2',
    'conv_tc3 k311 s11 256->256 @12x128x128 tile1x8x16 bn256 ln0 r1m p1 t1 st2',
    'conv_tc3 k311 s11 256->256 @12x128x128 tile1x8x16 bn256 ln0 r1m p1 t2 st2',
    'conv_tc3 k311 s11 256->256 @12x128x128 tile1x8x16 bn256 ln1 r0 p1 t1 st2',
    'conv_tc3 k311 s11 256->256 @12x128x128 tile1x8x16 bn256 ln1 r0 p1 t2 st2',
    'conv_tc3 k311 s11 256->256 @12x128x128 tile1x8x16 bn256 ln2 r1m p1 t1 st2',
    'conv_tc3 k311 s11 256->256 @12x128x128 tile1x8x16 bn256 ln2 r1m p1 t2 st2',
    'conv_tc3 k311 s11 256->256 @16x128x128 tile1x8x16 bn256 ln0 r1m p1 t0 st2 pad1.1',
    'conv_tc3 k311 s11 256->256 @16x128x128 tile1x8x16 bn256 ln1 r0 p1 t0 st2 pad1.1',
    'conv_tc3 k311 s11 256->256 @16x128x128 tile1x8x16 bn256 ln2 r1m p1 t0 st2 pad1.1',
    'conv_tc3 k311 s11 256->256 @18x128x128 tile1x8x16 bn256 ln0 r1m p1 t0 st2',
    'conv_tc3 k311 s11 256->256 @18x128x128 tile1x8x16 bn256 ln0 r1m p1 t1 st2',
    'conv_tc3 k311 s11 256->256 @18x128x128 tile1x8x16 bn256 ln0 r1m p1 t2 st2',
    'conv_tc3 k311 s11 256->256 @18x128x128 tile1x8x16 bn256 ln1 r0 p1 t0 st2',
    'conv_tc3 k311 s11 256->256 @18x128x128 tile1x8x16 bn256 ln1 r0 p1 t1 st2',
    'conv_tc3 k311 s11 256->256 @18x128x128 tile1x8x16 bn256 ln1 r0 p1 t2 st2',
    'conv_tc3 k311 s11 256->256 @18x128x128 tile1x8x16 bn256 ln2 r1m p1 t0 st2',
    'conv_tc3 k311 s11 256->256 @18x128x128 tile1x8x16 bn256 ln2 r1m p1 t1 st2',
    'conv_tc3 k311 s11 256->256 @18x128x128 tile1x8x16 bn256 ln2 r1m p1 t2 st2',
    'conv_tc3 k311 s11 256->256 @20x128x128 tile1x8x16 bn256 ln0 r1m p1 t1 st2',
    'conv_tc3 k311 s11 256->256 @20x128x128 tile1x8x16 bn256 ln1 r0 p1 t1 st2',
    'conv_tc3 k311 s11 256->256 @20x128x128 tile1x8x16 bn256 ln2 r1m p1 t1 st2',
    'conv_tc3 k311 s11 256->256 @2x128x128 tile1x8x16 bn256 ln0 r1m p1 t1 st2',
    'conv_tc3 k311 s11 256->256 @2x128x128 tile1x8x16 bn256 ln1 r0 p1 t1 st2',
    'conv_tc3 k311 s11 256->256 @2x128x128 tile1x8x16 bn256 ln2 r1m p1 t1 st2',
    'conv_tc3 k311 s11 256->256 @8x128x128 tile1x8x16 bn256 ln0 r1m p1 t0 st2 pad1.1',
    'conv_tc3 k311 s11 256->256 @8x128x128 tile1x8x16 bn256 ln0 r1m p1 t1 st2',
    'conv_tc3 k311 s11 256->256 @8x128x128 tile1x8x16 bn256 ln1 r0 p1 t0 st2 pad1.1',
    'conv_tc3 k311 s11 256->256 @8x128x128 tile1x8x16 bn256 ln1 r0 p1 t1 st2',
    'conv_tc3 k311 s11 256->256 @8x128x128 tile1x8x16 bn256 ln2 r1m p1 t0 st2 pad1.1',
    'conv_tc3 k311 s11 256->256 @8x128x128 tile1x8x16 bn256 ln2 r1m p1 t1 st2',
    'conv_tc3 k311 s11 512->512 @10x128x128 tile1x8x16 bn128 ln0 r0 p4 t0 st3',
    'conv_tc3 k311 s11 512->512 @10x128x128 tile1x8x16 bn128 ln0 r1m p4 t0 st3',
    'conv_tc3 k311 s11 512->512 @10x32x32 tile1x8x16 bn128 ln0 r0 p4 t0 st3',
    'conv_tc3 k311 s11 512->512 @10x32x32 tile1x8x16 bn128 ln0 r0 p4 t1 st3',
    'conv_tc3 k311 s11 512->512 @10x32x32 tile1x8x16 bn128 ln0 r1m p4 t0 st3',
    'conv_tc3 k311 s11 512->512 @10x32x32 tile1x8x16 bn128 ln0 r1m p4 t1 st3',
    'conv_tc3 k311 s11 512->512 @10x64x64 tile1x8x16 bn128 ln0 r0 p4 t1 st3',
    'conv_tc3 k311 s11 512->512 @10x64x64 tile1x8x16 bn128 ln0 r1m p4 t1 st3',
    'conv_tc3 k311 s11 512->512 @16x64x64 tile1x8x16 bn128 ln0 r0 p4 t0 st3 pad1.1',
    'conv_tc3 k311 s11 512->512 @16x64x64 tile1x8x16 bn128 ln0 r0 p4 t2 st3',
    'conv_tc3 k311 s11 512->512 @16x64x64 tile1x8x16 bn128 ln0 r1m p4 t0 st3 pad1.1',
    'conv_tc3 k311 s11 512->512 @16x64x64 tile1x8x16 bn128 ln0 r1m p4 t2 st3',
    'conv_tc3 k311 s11 512->512 @1x16x16 tile1x8x16 bn128 ln0 r0 p4 t1 st3',
    'conv_tc3 k311 s11 512->512 @1x16x16 tile1x8x16 bn128 ln0 r1m p4 t1 st3',
    'conv_tc3 k311 s11 512->512 @1x64x64 tile1x8x16 bn128 ln0 r0 p4 t1 st3',
    'conv_tc3 k311 s11 512->512 @1x64x64 tile1x8x16 bn128 ln0 r1m p4 t1 st3',
    'conv_tc3 k311 s11 512->512 @20x64x64 tile1x8x16 bn128 ln0 r0 p4 t0 st3',
    'conv_tc3 k311 s11 512->512 @20x64x64 tile1x8x16 bn128 ln0 r0 p4 t1 st3',
    'conv_tc3 k311 s11 512->512 @20x64x64 tile1x8x16 bn128 ln0 r1m p4 t0 st3',
    'conv_tc3 k311 s11 512->512 @20x64x64 tile1x8x16 bn128 ln0 r1m p4 t1 st3',
    'conv_tc3 k311 s11 512->512 @2x16x16 tile1x8x16 bn128 ln0 r0 p4 t1 st3',
    'conv_tc3 k311 s11 512->512 @2x16x16 tile1x8x16 bn128 ln0 r1m p4 t1 st3',
    'conv_tc3 k311 s11 512->512 @2x32x32 tile1x8x16 bn128 ln0 r0 p4 t2 st3',
    'conv_tc3 k311 s11 512->512 @2x32x32 tile1x8x16 bn128 ln0 r1m p4 t2 st3',
    'conv_tc3 k311 s11 512->512 @3x32x32 tile1x8x16 bn128 ln0 r0 p4 t1 st3',
    'conv_tc3 k311 s11 512->512 @3x32x32 tile1x8x16 bn128 ln0 r0 p4 t2 st3',
    'conv_tc3 k311 s11 512->512 @3x32x32 tile1x8x16 bn128 ln0 r1m p4 t1 st3',
    'conv_tc3 k311 s11 512->512 @3x32x32 tile1x8x16 bn128 ln0 r1m p4 t2 st3',
    'conv_tc3 k311 s11 512->512 @4x16x16 tile1x8x16 bn128 ln0 r0 p4 t0 st3 pad1.1',
    'conv_tc3 k311 s11 512->512 @4x16x16 tile1x8x16 bn128 ln0 r0 p4 t2 st3',
    'conv_tc3 k311 s11 512->512 @4x16x16 tile1x8x16 bn128 ln0 r1m p4 t0 st3 pad1.1',
    'conv_tc3 k311 s11 512->512 @4x16x16 tile1x8x16 bn128 ln0 r1m p4 t2 st3',
    'conv_tc3 k311 s11 512->512 @4x32x32 tile1x8x16 bn128 ln0 r0 p4 t0 st3 pad1.1',
    'conv_tc3 k311 s11 512->512 @4x32x32 tile1x8x16 bn128 ln0 r1m p4 t0 st3 pad1.1',
    'conv_tc3 k311 s11 512->512 @4x64x64 tile1x8x16 bn128 ln0 r0 p4 t0 st3 pad1.1',
    'conv_tc3 k311 s11 512->512 @4x64x64 tile1x8x16 bn128 ln0 r0 p4 t1 st3',
    'conv_tc3 k311 s11 512->512 @4x64x64 tile1x8x16 bn128 ln0 r1m p4 t0 st3 pad1.1',
    'conv_tc3 k311 s11 512->512 @4x64x64 tile1x8x16 bn128 ln0 r1m p4 t1 st3',
    'conv_tc3 k311 s11 512->512 @5x16x16 tile1x8x16 bn128 ln0 r0 p4 t0 st3',
    'conv_tc3 k311 s11 512->512 @5x16x16 tile1x8x16 bn128 ln0 r0 p4 t1 st3',
    'conv_tc3 k311 s11 512->512 @5x16x16 tile1x8x16 bn128 ln0 r0 p4 t2 st3',
    'conv_tc3 k311 s11 512->512 @5x16x16 tile1x8x16 bn128 ln0 r1m p4 t0 st3',
    'conv_tc3 k311 s11 512->512 @5x16x16 tile1x8x16 bn128 ln0 r1m p4 t1 st3',
    'conv_tc3 k311 s11 512->512 @5x16x16 tile1x8x16 bn128 ln0 r1m p4 t2 st3',
    'conv_tc3 k311 s11 512->512 @5x32x32 tile1x8x16 bn128 ln0 r0 p4 t1 st3',
    'conv_tc3 k311 s11 512->512 @5x32x32 tile1x8x16 bn128 ln0 r1m p4 t1 st3',
    'conv_tc3 k311 s11 512->512 @5x64x64 tile1x8x16 bn128 ln0 r0 p4 t1 st3',
    'conv_tc3 k311 s11 512->512 @5x64x64 tile1x8x16 bn128 ln0 r1m p4 t1 st3',
    'conv_tc3 k311 s11 512->512 @6x64x64 tile1x8x16 bn128 ln0 r0 p4 t1 st3',
    'conv_tc3 k311 s11 512->512 @6x64x64 tile1x8x16 bn128 ln0 r0 p4 t2 st3',
    'conv_tc3 k311 s11 512->512 @6x64x64 tile1x8x16 bn128 ln0 r1m p4 t1 st3',
    'conv_tc3 k311 s11 512->512 @6x64x64 tile1x8x16 bn128 ln0 r1m p4 t2 st3',
    'conv_tc3 k311 s11 512->512 @8x32x32 tile1x8x16 bn128 ln0 r0 p4 t0 st3 pad1.1',
    'conv_tc3 k311 s11 512->512 @8x32x32 tile1x8x16 bn128 ln0 r0 p4 t2 st3',
    'conv_tc3 k311 s11 512->512 @8x32x32 tile1x8x16 bn128 ln0 r1m p4 t0 st3 pad1.1',
    'conv_tc3 k311 s11 512->512 @8x32x32 tile1x8x16 bn128 ln0 r1m p4 t2 st3',
    'conv_tc3 k311 s11 512->512 @8x64x64 tile1x8x16 bn128 ln0 r0 p4 t0 st3 pad1.1',
    'conv_tc3 k311 s11 512->512 @8x64x64 tile1x8x16 bn128 ln0 r1m p4 t0 st3 pad1.1',
    'conv_tc3 k311 s11 512->512 @9x32x32 tile1x8x16 bn128 ln0 r0 p4 t0 st3',
    'conv_tc3 k311 s11 512->512 @9x32x32 tile1x8x16 bn128 ln0 r0 p4 t1 st3',
    'conv_tc3 k311 s11 512->512 @9x32x32 tile1x8x16 bn128 ln0 r0 p4 t2 st3',
    'conv_tc3 k311 s11 512->512 @9x32x32 tile1x8x16 bn128 ln0 r1m p4 t0 st3',
    'conv_tc3 k311 s11 512->512 @9x32x32 tile1x8x16 bn128 ln0 r1m p4 t1 st3',
    'conv_tc3 k311 s11 512->512 @9x32x32 tile1x8x16 bn128 ln0 r1m p4 t2 st3',
    'conv_tc3 k311 s11 512->512 @9x64x64 tile1x8x16 bn128 ln0 r0 p4 t0 st3',
    'conv_tc3 k311 s11 512->512 @9x64x64 tile1x8x16 bn128 ln0 r0 p4 t1 st3',
    'conv_tc3 k311 s11 512->512 @9x64x64 tile1x8x16 bn128 ln0 r0 p4 t2 st3',
    'conv_tc3 k311 s11 512->512 @9x64x64 tile1x8x16 bn128 ln0 r1m p4 t0 st3',
    'conv_tc3 k311 s11 512->512 @9x64x64 tile1x8x16 bn128 ln0 r1m p4 t1 st3',
    'conv_tc3 k311 s11 512->512 @9x64x64 tile1x8x16 bn128 ln0 r1m p4 t2 st3',
    'conv_tc3 k333 s11 128->3 @16x256x256 tile1x16x8 bn32 halo ln0 r0 p4 t0 st8 pad1.1',
    'conv_tc3 k333 s11 128->3 @16x256x256 tile1x16x8 bn32 halo ln0 r0 p4 t1 st8',
    'conv_tc3 k333 s11 128->3 @18x256x256 tile1x16x8 bn32 halo ln0 r0 p4 t1 st8',
    'conv_tc3 k333 s11 128->3 @18x256x256 tile1x16x8 bn32 halo ln0 r0 p4 t2 st8',
    'conv_tc3 k333 s11 128->3 @20x256x256 tile1x16x8 bn32 halo ln0 r0 p4 t1 st8',
    'conv_tc3 k333 s11 128->3 @24x256x256 tile1x16x8 bn32 halo ln0 r0 p4 t1 st8',
    'conv_tc3 k333 s11 128->3 @24x256x256 tile1x16x8 bn32 halo ln0 r0 p4 t2 st8',
    'conv_tc3 k333 s11 128->3 @4x256x256 tile1x16x8 bn32 halo ln0 r0 p4 t1 st8',
    'conv_tc3 k333 s11 256->256 @16x256x256 tile1x16x8 bn128 halo ln0 r1 p8 t1 st2',
    'conv_tc3 k333 s11 256->256 @20x256x256 tile1x16x8 bn128 halo ln0 r1 p8 t1 st2',
    'conv_tc3 k333 s11 256->256 @24x256x256 tile1x16x8 bn128 halo ln0 r1 p8 t1 st2',
    'conv_tc3 k333 s11 256->256 @24x256x256 tile1x16x8 bn128 halo ln0 r1 p8 t2 st2',
    'conv_tc3 k333 s11 512->16 @1x32x32 tile1x16x8 bn32 halo ln0 r0 p8 t1 st7',
    'conv_tc3 k333 s11 512->16 @5x32x32 tile1x16x8 bn32 halo ln0 r0 p8 t0 st7',
    'conv_tc3 k333 s11 512->16 @8x32x32 tile1x16x8 bn32 halo ln0 r0 p8 t2 st7',
    'conv_tc3 k333 s11 512->16 @9x32x32 tile1x16x8 bn32 halo ln0 r0 p8 t0 st7',
    'conv_tc3 k333 s11 512->16 @9x32x32 tile1x16x8 bn32 halo ln0 r0 p8 t1 st7',
    'conv_tc3 k333 s11 512->32 @1x16x16 tile1x16x8 bn32 halo ln0 r0 p8 t1 st7',
    'conv_tc3 k333 s11 512->32 @4x16x16 tile1x16x8 bn32 halo ln0 r0 p8 t0 st7 pad1.1',
    'conv_tc3 k333 s11 512->32 @4x16x16 tile1x16x8 bn32 halo ln0 r0 p8 t2 st7',
    'conv_tc3 k333 s11 512->32 @4x32x32 tile1x16x8 bn32 halo ln0 r0 p8 t0 st7 pad1.1',
    'conv_tc3 k333 s11 512->32 @5x16x16 tile1x16x8 bn32 halo ln0 r0 p8 t1 st7',
    'conv_tc3 k333 s11 512->32 @5x32x32 tile1x16x8 bn32 halo ln0 r0 p8 t0 st7',
    'conv_tc3 k333 s11 512->32 @5x32x32 tile1x16x8 bn32 halo ln0 r0 p8 t1 st7',
    'conv_tc3 k333 s11 512->4 @5x32x32 tile1x16x8 bn32 halo ln0 r0 p8 t0 st7',
    'conv_tc3 k333 s11 512->5 @1x32x32 tile1x16x8 bn32 halo ln0 r0 p8 t1 st7',
    'conv_tc3 k333 s11 512->5 @2x32x32 tile1x16x8 bn32 halo ln0 r0 p8 t2 st7',
    'conv_tc3 k333 s11 512->5 @3x32x32 tile1x16x8 bn32 halo ln0 r0 p8 t1 st7',
    'conv_tc3 k333 s11 512->5 @4x32x32 tile1x16x8 bn32 halo ln0 r0 p8 t2 st7',
    'conv_tc3 k333 s11 512->5 @5x32x32 tile1x16x8 bn32 halo ln0 r0 p8 t1 st7',
    'conv_tc3 k333 s11 512->512 @10x128x128 tile1x16x8 bn64 halo ln0 r1 p8 t1 st4',
    'conv_tc3 k333 s11 512->512 @12x128x128 tile1x16x8 bn64 halo ln0 r1 p8 t1 st4',
    'conv_tc3 k333 s11 512->512 @12x128x128 tile1x16x8 bn64 halo ln0 r1 p8 t2 st4',
    'conv_tc3 k333 s11 512->512 @16x128x128 tile1x16x8 bn64 halo ln0 r1 p8 t2 st4',
    'conv_tc3 k333 s11 512->512 @18x128x128 tile1x16x8 bn64 halo ln0 r1 p8 t1 st4',
    'conv_tc3 k333 s11 512->512 @18x128x128 tile1x16x8 bn64 halo ln0 r1 p8 t2 st4',
    'conv_tc3 k333 s11 512->512 @1x16x16 tile1x16x8 bn64 halo ln0 r0 p8 t1 st4',
    'conv_tc3 k333 s11 512->512 @1x16x16 tile1x16x8 bn64 halo ln0 r1m p8 t1 st4',
    'conv_tc3 k333 s11 512->512 @2x16x16 tile1x16x8 bn64 halo ln0 r0 p8 t1 st4',
    'conv_tc3 k333 s11 512->512 @2x16x16 tile1x16x8 bn64 halo ln0 r1m p8 t1 st4',
    'conv_tc3 k333 s11 512->512 @2x32x32 tile1x16x8 bn64 halo ln0 r0 p8 t2 st4',
    'conv_tc3 k333 s11 512->512 @2x32x32 tile1x16x8 bn64 halo ln0 r1m p8 t2 st4',
    'conv_tc3 k333 s11 512->512 @3x32x32 tile1x16x8 bn64 halo ln0 r0 p8 t1 st4',
    'conv_tc3 k333 s11 512->512 @3x32x32 tile1x16x8 bn64 halo ln0 r0 p8 t2 st4',
    'conv_tc3 k333 s11 512->512 @3x32x32 tile1x16x8 bn64 halo ln0 r1m p8 t1 st4',
    'conv_tc3 k333 s11 512->512 @3x32x32 tile1x16x8 bn64 halo ln0 r1m p8 t2 st4',
    'conv_tc3 k333 s11 512->512 @4x16x16 tile1x16x8 bn64 halo ln0 r0 p8 t0 st4 pad1.1',
    'conv_tc3 k333 s11 512->512 @4x16x16 tile1x16x8 bn64 halo ln0 r0 p8 t2 st4',
    'conv_tc3 k333 s11 512->512 @4x16x16 tile1x16x8 bn64 halo ln0 r1m p8 t0 st4 pad1.1',
    'conv_tc3 k333 s11 512->512 @4x16x16 tile1x16x8 bn64 halo ln0 r1m p8 t2 st4',
    'conv_tc3 k333 s11 512->512 @4x32x32 tile1x16x8 bn64 halo ln0 r0 p8 t0 st4 pad1.1',
    'conv_tc3 k333 s11 512->512 @4x32x32 tile1x16x8 bn64 halo ln0 r1m p8 t0 st4 pad1.1',
    'conv_tc3 k333 s11 512->512 @4x64x64 tile1x16x8 bn64 halo ln0 r1 p8 t1 st4',
    'conv_tc3 k333 s11 512->512 @4x64x64 tile1x16x8 bn64 halo ln0 r1 p8 t2 st4',
    'conv_tc3 k333 s11 512->512 @5x16x16 tile1x16x8 bn64 halo ln0 r0 p8 t0 st4',
    'conv_tc3 k333 s11 512->512 @5x16x16 tile1x16x8 bn64 halo ln0 r0 p8 t1 st4',
    'conv_tc3 k333 s11 512->512 @5x16x16 tile1x16x8 bn64 halo ln0 r0 p8 t2 st4',
    'conv_tc3 k333 s11 512->512 @5x16x16 tile1x16x8 bn64 halo ln0 r1m p8 t0 st4',
    'conv_tc3 k333 s11 512->512 @5x16x16 tile1x16x8 bn64 halo ln0 r1m p8 t1 st4',
    'conv_tc3 k333 s11 512->512 @5x16x16 tile1x16x8 bn64 halo ln0 r1m p8 t2 st4',
    'conv_tc3 k333 s11 512->512 @5x32x32 tile1x16x8 bn64 halo ln0 r0 p8 t1 st4',
    'conv_tc3 k333 s11 512->512 @5x32x32 tile1x16x8 bn64 halo ln0 r1m p8 t1 st4',
    'conv_tc3 k333 s11 512->512 @5x64x64 tile1x16x8 bn64 halo ln0 r0 p8 t0 st4',
    'conv_tc3 k333 s11 512->512 @5x64x64 tile1x16x8 bn64 halo ln0 r1m p8 t0 st4',
    'conv_tc3 k333 s11 512->512 @6x64x64 tile1x16x8 bn64 halo ln0 r1 p8 t1 st4',
    'conv_tc3 k333 s11 512->512 @6x64x64 tile1x16x8 bn64 halo ln0 r1 p8 t2 st4',
    'conv_tc3 k333 s11 512->512 @8x128x128 tile1x16x8 bn64 halo ln0 r1 p8 t1 st4',
    'conv_tc3 k333 s11 512->512 @8x32x32 tile1x16x8 bn64 halo ln0 r0 p8 t2 st4',
    'conv_tc3 k333 s11 512->512 @8x32x32 tile1x16x8 bn64 halo ln0 r1m p8 t2 st4',
    'conv_tc3 k333 s11 512->512 @9x32x32 tile1x16x8 bn64 halo ln0 r0 p8 t0 st4',
    'conv_tc3 k333 s11 512->512 @9x32x32 tile1x16x8 bn64 halo ln0 r0 p8 t1 st4',
    'conv_tc3 k333 s11 512->512 @9x32x32 tile1x16x8 bn64 halo ln0 r0 p8 t2 st4',
    'conv_tc3 k333 s11 512->512 @9x32x32 tile1x16x8 bn64 halo ln0 r1m p8 t0 st4',
    'conv_tc3 k333 s11 512->512 @9x32x32 tile1x16x8 bn64 halo ln0 r1m p8 t1 st4',
    'conv_tc3 k333 s11 512->512 @9x32x32 tile1x16x8 bn64 halo ln0 r1m p8 t2 st4',
    'conv_tc3 k333 s11 512->6 @1x16x16 tile1x16x8 bn32 halo ln0 r0 p8 t1 st7',
    'conv_tc3 k333 s11 512->6 @4x16x16 tile1x16x8 bn32 halo ln0 r0 p8 t0 st7 pad1.1',
    'conv_tc3 k333 s11 512->6 @4x16x16 tile1x16x8 bn32 halo ln0 r0 p8 t2 st7',
    'conv_tc3 k333 s11 512->6 @4x32x32 tile1x16x8 bn32 halo ln0 r0 p8 t0 st7 pad1.1',
    'conv_tc3 k333 s11 512->6 @5x16x16 tile1x16x8 bn32 halo ln0 r0 p8 t0 st7',
    'conv_tc3 k333 s11 512->6 @5x16x16 tile1x16x8 bn32 halo ln0 r0 p8 t1 st7',
    'conv_tc3 k333 s11 512->6 @5x32x32 tile1x16x8 bn32 halo ln0 r0 p8 t0 st7',
    'conv_tc3 k333 s11 512->8 @1x32x32 tile1x16x8 bn32 halo ln0 r0 p8 t1 st7',
    'conv_tc3 k333 s11 512->8 @4x16x16 tile1x16x8 bn32 halo ln0 r0 p8 t0 st7 pad1.1',
    'conv_tc3 k333 s11 512->8 @4x32x32 tile1x16x8 bn32 halo ln0 r0 p8 t0 st7 pad1.1',
    'conv_tc3 k333 s11 512->8 @4x32x32 tile1x16x8 bn32 halo ln0 r0 p8 t2 st7',
    'conv_tc3 k333 s11 512->8 @5x16x16 tile1x16x8 bn32 halo ln0 r0 p8 t0 st7',
    'conv_tc3 k333 s11 512->8 @5x32x32 tile1x16x8 bn32 halo ln0 r0 p8 t1 st7',
    'conv_tc3 k333 s11 512->8 @5x64x64 tile1x16x8 bn32 halo ln0 r0 p8 t0 st7',
    'conv_tc3 k333 s21 128->128 @12x128x128 tile1x16x8 bn128 halo ln2 r3 p4 t1 st2',
    'conv_tc3 k333 s21 128->128 @4x128x128 tile1x16x8 bn128 halo ln2 r3 p4 t1 st2',
    'conv_tc3 k333 s21 128->128 @8x128x128 tile1x16x8 bn128 halo ln2 r3 p4 t2 st2',
    'conv_tc3 k333 s21 256->256 @10x128x128 tile1x16x8 bn128 halo ln0 r3 p8 t0 st2',
    'conv_tc3 k333 s21 256->256 @10x64x64 tile1x16x8 bn128 halo ln0 r3 p8 t1 st2',
    'conv_tc3 k333 s21 256->256 @1x64x64 tile1x16x8 bn128 halo ln0 r3 p8 t1 st2',
    'conv_tc3 k333 s21 256->256 @4x64x64 tile1x16x8 bn128 halo ln0 r3 p8 t2 st2',
    'conv_tc3 k333 s21 256->256 @6x64x64 tile1x16x8 bn128 halo ln0 r3 p8 t1 st2',
    'conv_tc3 k333 s21 256->256 @8x64x64 tile1x16x8 bn128 halo ln0 r3 p8 t0 st2 pad0.1 pool1',
    'conv_tc3 k333 s21 256->256 @9x64x64 tile1x16x8 bn128 halo ln0 r3 p8 t0 st2',
    'conv_tc3 k333 s21 256->256 @9x64x64 tile1x16x8 bn128 halo ln0 r3 p8 t1 st2',
    'conv_tc3 k333 s21 512->512 @10x32x32 tile1x16x8 bn64 halo ln0 r3 p8 t0 st4',
    'conv_tc3 k333 s21 512->512 @10x32x32 tile1x16x8 bn64 halo ln0 r3 p8 t1 st4',
    'conv_tc3 k333 s21 512->512 @1x16x16 tile1x16x8 bn64 halo ln0 r3 p8 t1 st4',
    'conv_tc3 k333 s21 512->512 @2x32x32 tile1x16x8 bn64 halo ln0 r3 p8 t1 st4',
    'conv_tc3 k333 s21 512->512 @2x32x32 tile1x16x8 bn64 halo ln0 r3 p8 t2 st4',
    'conv_tc3 k333 s21 512->512 @3x32x32 tile1x16x8 bn64 halo ln0 r3 p8 t1 st4',
    'conv_tc3 k333 s21 512->512 @4x16x16 tile1x16x8 bn64 halo ln0 r3 p8 t0 st4 pad0.1 pool1',
    'conv_tc3 k333 s21 512->512 @4x16x16 tile1x16x8 bn64 halo ln0 r3 p8 t2 st4',
    'conv_tc3 k333 s21 512->512 @4x32x32 tile1x16x8 bn64 halo ln0 r3 p8 t0 st4 pad0.1 pool1',
    'conv_tc3 k333 s21 512->512 @5x16x16 tile1x16x8 bn64 halo ln0 r3 p8 t0 st4',
    'conv_tc3 k333 s21 512->512 @5x16x16 tile1x16x8 bn64 halo ln0 r3 p8 t1 st4',
    'conv_tc3 k333 s21 512->512 @5x32x32 tile1x16x8 bn64 halo ln0 r3 p8 t1 st4',
    'conv_tc3 k333 s21 512->512 @5x64x64 tile1x16x8 bn64 halo ln0 r3 p8 t0 st4',
    'conv_tc3 k333 s21 512->512 @8x32x32 tile1x16x8 bn64 halo ln0 r3 p8 t0 st4 pad0.1 pool1',
    'conv_tc3 k333 s21 512->512 @8x32x32 tile1x16x8 bn64 halo ln0 r3 p8 t2 st4',
    'tblock_tc strip 1x128 T18 ln_out0',
    'tblock_tc strip 1x128 T18 ln_out1',
]


def zoo_forward_keys():
    """{case id: sorted plan keys} of one bf16 and one exact forward of each MODEL_CASES entry"""
    from gpu_util import plan_keys
    out = {}
    for case in MODEL_CASES:
        name, tiled = case
        model, _, x = zoo_model(name, tiled)
        xd = x.cuda()
        keys = set()
        for prec in ("bf16", "exact"):
            model.precision = prec
            torch.manual_seed(NOISE_SEED)
            with torch.no_grad():
                _, k = plan_keys(lambda: model(xd))
            assert k, (name, prec)
            keys |= set(k)
        out[case_id(case)] = sorted(keys)
        del model, xd
        gc.collect()
        torch.cuda.empty_cache()
    return out


def test_zoo_table_is_well_formed():
    assert len(set(ZOO_PLAN_TABLE)) == len(ZOO_PLAN_TABLE) and not set(ZOO_PLAN_TABLE) & set(PLAN_TABLE)
    assert ZOO_PLAN_TABLE == sorted(ZOO_PLAN_TABLE)
    for key in ZOO_PLAN_TABLE:
        entry_of(parse(key))


def test_zoo_forward_keys_are_in_tables():
    table = set(PLAN_TABLE) | set(ZOO_PLAN_TABLE)
    launched, missing = set(), {}
    for cid, keys in zoo_forward_keys().items():
        launched |= set(keys)
        miss = sorted(set(keys) - table)
        print(f"[{cid}] {len(keys)} plan keys, {len(miss)} in neither table")
        if miss:
            missing[cid] = miss
    stale = sorted(set(ZOO_PLAN_TABLE) - launched)
    assert not missing and not stale, ("plan keys without a case:\n" + "\n".join(f"  {c}: {k}" for c, ks in missing.items() for k in ks)
                                       + "\nstale ZOO_PLAN_TABLE keys:\n" + "\n".join(f"  {k}" for k in stale))


@pytest.mark.parametrize("key", ZOO_PLAN_TABLE)
def test_zoo_plan_case(key):
    check_case(key, prec_of(parse(key)), run_case(key))


if __name__ == "__main__":
    # regenerate ZOO_PLAN_TABLE on an H100, from the repository root: PYTHONPATH=. python tests/test_gpu_zoo.py
    keys = sorted(set(k for ks in zoo_forward_keys().values() for k in ks) - set(PLAN_TABLE))
    print("ZOO_PLAN_TABLE = [")
    for k in keys:
        print(f"    {k!r},")
    print("]")
