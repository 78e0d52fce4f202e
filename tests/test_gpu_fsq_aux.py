"""-m gpu: the FSQ auxiliary loss on the device (csrc/fsq_aux.cu through FSQRegularizer / both engines) against the values of
the unmodified reference stored in tests/golden/fsq_aux and against the fp64 oracle (oracle/fsq_aux_oracle.py)."""
import ctypes as C
import json

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from conftest import load_golden, synth_inputs, synth_weights  # noqa: E402
from test_fsq_aux_cpu import CASES, COMPONENTS, load_aux  # noqa: E402

SHIPPED = dict(entropy_loss_weight=0.1, entropy_loss_annealing_steps=2000, entropy_loss_annealing_factor=3,
               commitment_loss_weight=0.25)


def reg_for(levels, **kw):
    from vidtok_b200.engine import FSQRegularizer
    return FSQRegularizer(list(levels), **(kw or SHIPPED)).cuda()


def device_components(reg, hs, world_size=None, avg_sum=None):
    """partials of each segment in hs, finalize -> ({component: [per segment]}, aux_loss)"""
    parts = [reg.aux_partials(h.cuda()) for h in hs]
    stats = torch.cat([p[0] for p in parts])
    avg = torch.cat([p[1] for p in parts]) if avg_sum is None else avg_sum
    comp = torch.empty((len(hs), 4), dtype=torch.float32, device="cuda")
    aux = reg.aux_finalize(stats, avg, world_size=world_size or 1, components=comp)
    comp = comp.cpu()
    return {k: [float(comp[s, i]) for s in range(len(hs))] for i, k in enumerate(COMPONENTS)}, float(aux)


def bound(meta, k):
    return max(1e-5, 4.0 * meta["deviation"][k])


def rel(a, b):
    return abs(a - b) / max(abs(b), 1e-12)


@pytest.mark.parametrize("case", [c for c in CASES if load_aux(c)[1]["kind"] == "single"])
def test_partials_and_finalize_match_reference(case):
    d, meta = load_aux(case)
    got, aux = device_components(reg_for(meta["levels"]), [torch.from_numpy(d["h"])])
    o = meta["oracle"]
    for k in COMPONENTS[:3]:
        g = got[k][0]
        print(f"{case} {k}: device {g:.9g} reference {meta['reference'][k]:.9g} oracle {o[k]:.9g}")
        assert rel(g, o[k]) <= bound(meta, k), (k, g, o[k])
        assert rel(g, meta["reference"][k]) <= bound(meta, k), (k, g, meta["reference"][k])
    # aux_loss = (pse - cbe) * 0.3 + commit * 0.25 can cancel to far below its terms (syn_peaked_8888: -0.0019 from terms of
    # about 1), so its error is bounded relative to the size of the terms it sums
    scale = 0.3 * (abs(o["per_sample_entropy"]) + abs(o["codebook_entropy"])) + 0.25 * abs(o["commit_loss"])
    for name, want in (("oracle", o["aux_loss"]), ("reference", meta["reference"]["aux_loss"])):
        err = abs(got["aux_loss"][0] - want) / scale
        print(f"{case} aux_loss: device {got['aux_loss'][0]:.9g} {name} {want:.9g} error / term scale {err:.3e}")
        assert err <= max(1e-5, 4.0 * meta["deviation"]["aux_loss"] * abs(want) / scale), (name, err)
    assert aux == got["aux_loss"][0]


def test_chunked_segments_match_tile_encode_reference():
    d, meta = load_aux("tiled_tiny_fsq_v11_tiled")
    _, aux = device_components(reg_for(meta["levels"]), [torch.from_numpy(d[f"h{i}"]) for i in range(meta["n_chunks"])])
    assert rel(aux, meta["reference"]["aux_loss"]) <= bound(meta, "aux_loss")
    assert rel(aux, meta["oracle"]["aux_loss"]) <= bound(meta, "aux_loss")


def test_distributed_mean_of_two_halves():
    """all_reduce(avg_prob) / world_size (regularizers.py:49-59,240): the halves' avg_prob summed, then each half finalized
    with world_size 2, reproduces the two-rank gloo run of the reference."""
    d, meta = load_aux("dist2_88888")
    reg = reg_for(meta["levels"])
    h = torch.from_numpy(d["h"])
    halves = [h[:2], h[2:]]
    parts = [reg.aux_partials(x.cuda()) for x in halves]
    avg_sum = parts[0][1] + parts[1][1]
    for r in range(2):
        comp = torch.empty((1, 4), dtype=torch.float32, device="cuda")
        reg.aux_finalize(parts[r][0], avg_sum.clone(), world_size=2, components=comp)
        for i, k in enumerate(COMPONENTS):
            assert rel(float(comp[0, i]), meta["reference_ranks"][r][k]) <= bound(meta, k), (r, k)


def test_two_runs_are_bit_identical():
    for case in ("syn_flat_888888", "syn_encoder_88888", "fix_cfg1_fsq_488_32768"):
        d, meta = load_aux(case)
        reg = reg_for(meta["levels"])
        h = torch.from_numpy(d["h"]).cuda()
        a, b = reg.aux_loss(h), reg.aux_loss(h)
        sa, pa = reg.aux_partials(h)
        sb, pb = reg.aux_partials(h)
        assert torch.equal(a, b) and torch.equal(sa, sb) and torch.equal(pa, pb), case


def test_unsupported_level_lists_are_rejected():
    from vidtok_b200 import _native as N
    lib = N.lib()
    for levels in ([8] * 8, [1, 8, 8], [300, 2]):
        arr = (C.c_int32 * len(levels))(*levels)
        assert lib.vt_fsq_aux_workspace_bytes(len(levels), arr, 1024) == -1
        assert b"FSQ aux loss" in lib.vt_last_error()


def _fsq488(levels=(8, 8, 8, 8, 8), **reg_kw):
    import bench
    from vidtok_b200.compat_util import instantiate_from_config
    from vidtok_b200.synth import synth_state_dict
    cfg = bench.model_cfg(bench.CONFIGS["fsq488"])
    cfg["params"]["regularizer_config"]["params"] = dict(levels=list(levels), **(reg_kw or SHIPPED))
    model = instantiate_from_config(cfg)
    model.load_state_dict(synth_state_dict({k: tuple(v.shape) for k, v in model.state_dict().items()}, seed=0))
    return model.cuda().eval()


def test_production_batch_against_oracle():
    """fsq488: 8 clips 17x256x256 in exact mode (40 960 tokens, 32 768 codes) against the fp64 oracle on the engine's own h."""
    from oracle.fsq_aux_oracle import fsq_aux_loss
    from vidtok_b200.synth import synth_clip
    model = _fsq488()
    model.precision = "exact"
    x = synth_clip(8, 17, 256, 256, seed=1234).cuda()
    with torch.no_grad():
        h = model.encoder(x)
        _, log = model.encode(x, return_reg_log=True)
    assert h.shape == (8, 5, 5, 32, 32)
    ora = fsq_aux_loss(h, [8] * 5, **SHIPPED)
    got = float(model.regularization.aux_loss(h))
    print(f"fsq488 aux: device {got:.9g} oracle {float(ora['aux_loss']):.9g} rel {rel(got, float(ora['aux_loss'])):.3e}")
    assert rel(got, float(ora["aux_loss"])) <= 1e-5
    assert float(log["aux_loss"]) == got   # encode's reg_log is the same computation on the same h


def test_peak_memory_for_262144_codes():
    reg = reg_for([8] * 6)
    h = (torch.randn((8, 6, 5, 32, 32), generator=torch.Generator().manual_seed(3)) * 0.5).cuda()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.max_memory_allocated()
    aux = reg.aux_loss(h)
    torch.cuda.synchronize()
    grow = torch.cuda.max_memory_allocated() - base
    print(f"262144 codes, 40960 tokens: aux {float(aux):.6g}, peak memory growth {grow / 2**20:.1f} MiB")
    assert grow < 32 * 2**20, grow   # the materialised form needs 2 x 43 GB


def _model_for(case):
    from test_gpu_model import build_model
    d, meta = load_golden(case)
    sd, x = synth_weights(meta, d), synth_inputs(meta, d)
    return d, meta, build_model(meta, sd), x


# exact mode's latent error (<= 3e-5) moves the softmax logits 2 * 100 * |dz| * |c|: measured below, bounded loosely
E2E_BOUND = 2e-3


@pytest.mark.parametrize("case", ["tiny_fsq_v10", "mid_fsq_v10", "tiny_fsq_nc", "tiny_fsq_888_v11", "cfg1_fsq_488_32768"])
def test_engine_forward_aux_loss(case):
    _, meta = load_aux("fix_" + case)
    d, gmeta, model, x = _model_for(case)
    model.precision = "exact"
    with torch.no_grad():
        _, _, log = model(x.cuda())
    got, want = float(log["aux_loss"]), meta["reference"]["aux_loss"]
    assert log["aux_loss"].is_cuda and log["aux_loss"].dim() == 0
    print(f"{case}: forward aux_loss {got:.9g} reference {want:.9g} relative error {rel(got, want):.3e}")
    assert rel(got, want) <= E2E_BOUND


def test_tile_encode_aux_loss_device_and_host_inputs():
    _, meta = load_aux("tiled_tiny_fsq_v11_tiled")
    d, gmeta, model, x = _model_for("tiny_fsq_v11_tiled")
    model.precision = "exact"
    with torch.no_grad():
        _, log_dev = model.encode(x.cuda(), return_reg_log=True)
        _, log_host = model.encode(x.pin_memory(), return_reg_log=True)
    assert torch.equal(log_dev["aux_loss"], log_host["aux_loss"])
    got, want = float(log_dev["aux_loss"]), meta["reference"]["aux_loss"]
    print(f"tile_encode aux_loss {got:.9g} reference {want:.9g} relative error {rel(got, want):.3e}")
    assert rel(got, want) <= E2E_BOUND


def test_zero_weights_give_zero_and_launch_no_aux_kernel():
    from test_gpu_model import profiled_forward
    from vidtok_b200 import _native as N  # noqa: F401
    d, meta, model, x = _model_for("tiny_fsq_v10")
    model.regularization.entropy_loss_weight = 0.0
    model.regularization.commitment_loss_weight = 0.0
    _, _, log, launches = profiled_forward(model, x.cuda(), 0)
    assert float(log["aux_loss"]) == 0.0
    assert not any(k.startswith("fsq_aux") for k in launches), launches
    model.regularization.entropy_loss_weight = 0.1
    _, _, log, launches = profiled_forward(model, x.cuda(), 0)
    assert float(log["aux_loss"]) != 0.0
    assert {"fsq_aux_tokens", "fsq_aux_avgprob", "fsq_aux_reduce", "fsq_aux_finish"} <= set(launches), launches
