"""-m gpu: one long video as shards in one batch (encode_sharded / decode_sharded) against tile_encode / tile_decode: the
latents, FSQ indices, FSQ aux_loss and decoded frames are bit-identical and kl_loss agrees to 1e-6 in every precision mode,
for 1, 2, 3 and 5 shards, with videos long enough that every shard past the first warms up and the last one owns an
unequal remainder; over two ranks when the machine has two GPUs."""
import gc

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _release_models():
    """Each model parks the chunk caches of every batch size it ran in its own pool: return them between tests."""
    yield
    gc.collect()
    torch.cuda.empty_cache()

from conftest import load_golden, resolved_model_cfg, synth_weights  # noqa: E402


def _model(case, mode):
    from vidtok_b200.compat_util import instantiate_from_config
    d, meta = load_golden(case)
    model = instantiate_from_config(resolved_model_cfg(meta))
    missing, unexpected = model.load_state_dict(synth_weights(meta, d), strict=False)
    assert not missing and not unexpected
    model = model.to("cuda").eval()
    model.precision = mode
    return model


def _video(T, seed, H=32):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand((1, 3, T, H, H), generator=g) * 2 - 1)


@pytest.mark.parametrize("mode", ["bf16", "fma", "exact"])
@pytest.mark.parametrize("case", ["tiny_kl_v11_tiled", "tiny_fsq_v11_tiled"])
def test_encode_sharded_equals_tile_encode(case, mode):
    from vidtok_b200.longvideo import encode_sharded
    model = _model(case, mode)
    x = _video(1 + 16 * 14 + 5, 1).cuda()     # 15 chunks after the first frame, a short last one
    torch.manual_seed(7)
    z_ref, log_ref = model.tile_encode(x)
    for S in (1, 2, 3, 5):
        torch.manual_seed(7)
        z, log = encode_sharded(model, x, S)
        _same_encode(z, log, z_ref, log_ref, S)


def _same_encode(z, log, z_ref, log_ref, S):
    assert z.dtype == z_ref.dtype and torch.equal(z, z_ref), (S, (z.float() - z_ref.float()).abs().max())
    assert set(log) == set(log_ref), (set(log), set(log_ref))
    if "indices" in log_ref:
        assert torch.equal(log["indices"], log_ref["indices"]), S
        assert torch.equal(log["aux_loss"], log_ref["aux_loss"]), (S, float(log["aux_loss"]), float(log_ref["aux_loss"]))
    else:
        a, b = float(log["kl_loss"]), float(log_ref["kl_loss"])
        assert abs(a - b) <= 1e-6 * abs(b), (S, a, b)


@pytest.mark.parametrize("mode", ["bf16", "fma", "exact"])
@pytest.mark.parametrize("overlap", [False, True])
@pytest.mark.parametrize("case", ["tiny_kl_v11_tiled", "tiny_fsq_v11_tiled"])
def test_decode_sharded_equals_tile_decode(case, overlap, mode):
    from vidtok_b200.longvideo import decode_sharded
    model = _model(case, mode)
    model.t_chunk_dec, model.use_overlap = 4, overlap
    g = torch.Generator().manual_seed(3)
    z = torch.randn((1, model.spec.z_channels, 1 + 4 * 20 + 2, 4, 4), generator=g).cuda()   # 21 chunks, a short last one
    y_ref = model.tile_decode(z)
    for S in (1, 2, 3, 5):
        y = decode_sharded(model, z, S)
        assert torch.equal(y, y_ref), (S, (y - y_ref).abs().max())


@pytest.mark.parametrize("case", ["tiny_kl_v11_tiled", "tiny_fsq_v11_tiled"])
def test_autocast_returns_fp32_like_the_tile_paths(case):
    from vidtok_b200.longvideo import decode_sharded, encode_sharded
    model = _model(case, None)
    model.t_chunk_dec, model.use_overlap = 4, True
    x = _video(1 + 16 * 14 + 5, 2).cuda()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        torch.manual_seed(7)
        z_ref, log_ref = model.tile_encode(x)
        torch.manual_seed(7)
        z, log = encode_sharded(model, x, 2)
        _same_encode(z, log, z_ref, log_ref, 2)
        zl = torch.randn((1, model.spec.z_channels, 1 + 4 * 20 + 2, 4, 4), generator=torch.Generator().manual_seed(3)).cuda()
        y_ref = model.tile_decode(zl)
        y = decode_sharded(model, zl, 3)
    assert y.dtype == y_ref.dtype == torch.float32 and torch.equal(y, y_ref)


def _kl488(mode):
    import gzip
    import json
    import os
    from vidtok_b200.compat_util import instantiate_from_config
    from vidtok_b200.synth import synth_state_dict
    zoo = json.load(gzip.open(os.path.join(os.path.dirname(__file__), "golden", "zoo_manifest.json.gz"), "rt"))
    rec = zoo["vidtok_v1_1/vidtok_kl_causal_488_4chn_v1_1.yaml"]
    model = instantiate_from_config(rec["model"])
    model.load_state_dict(synth_state_dict({k: tuple(v) for k, v in rec["shapes"].items()}, seed=0), strict=False)
    model = model.to("cuda").eval()
    model.precision, model.use_overlap = mode, True
    return model


@pytest.mark.parametrize("mode", ["bf16", "fma", "exact"])
def test_kl488_host_video(mode):
    """kl_causal_488_4chn_v1_1 at 256^2 with synthetic weights: the video in pinned host memory, the decoded frames into a
    pinned host tensor."""
    from vidtok_b200.longvideo import decode_sharded, encode_sharded
    model = _kl488(mode)
    x = _video(1 + 16 * 20 + 7, 5, H=256).pin_memory()
    torch.manual_seed(11)
    z_ref, log_ref = model.tile_encode(x)
    y_ref = model.tile_decode(z_ref)
    for S in (1, 2, 3, 5):
        torch.manual_seed(11)
        z, log = encode_sharded(model, x, S)
        _same_encode(z, log, z_ref, log_ref, S)
        out = torch.empty(tuple(y_ref.shape), dtype=torch.float32).pin_memory()
        assert decode_sharded(model, z_ref, S, out=out) is out
        assert torch.equal(out, y_ref.cpu()), S


def _two_ranks(rank, path, result):
    import torch.distributed as dist
    from vidtok_b200.longvideo import decode_sharded, encode_sharded
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", init_method="file://" + path, rank=rank, world_size=2)
    try:
        model = _kl488("bf16")
        x = _video(1 + 16 * 20 + 7, 5, H=256)
        torch.manual_seed(11)
        z, log = encode_sharded(model, x.cuda(), 4)
        y, (g0, g1) = decode_sharded(model, z, 4)
        torch.save({"z": z.cpu(), "kl": log["kl_loss"].cpu(), "y": y.cpu(), "range": (g0, g1)}, f"{result}.{rank}")
    finally:
        dist.destroy_process_group()


def test_two_ranks():
    """Each rank's owned frames equal the slice of the one-GPU tile_decode; the gathered latents equal tile_encode's."""
    import os
    import tempfile
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs: this machine has fewer, so the rank path is not run here")
    import torch.multiprocessing as mp
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_two_ranks, args=(os.path.join(d, "store"), os.path.join(d, "out")), nprocs=2, join=True)
        res = [torch.load(os.path.join(d, f"out.{r}")) for r in range(2)]
    model = _kl488("bf16")
    x = _video(1 + 16 * 20 + 7, 5, H=256).cuda()
    torch.manual_seed(11)
    z_ref, log_ref = model.tile_encode(x)
    y_ref = model.tile_decode(z_ref).cpu()
    assert res[0]["range"][0] == 0 and res[0]["range"][1] == res[1]["range"][0] and res[1]["range"][1] == y_ref.shape[2]
    for r in res:
        assert torch.equal(r["z"], z_ref.cpu())
        assert abs(float(r["kl"]) - float(log_ref["kl_loss"])) <= 1e-6 * abs(float(log_ref["kl_loss"]))
        g0, g1 = r["range"]
        assert torch.equal(r["y"], y_ref[:, :, g0:g1])
