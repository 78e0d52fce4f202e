"""Host side of LPIPS (vidtok_b200.metrics.LPIPS, vt_lpips_*): the loader's key tables and refusals, the pass-size rule, the
workspace query with its widened products, argument errors that launch nothing, the grouping identity of the evaluation
script, and (where the reference checkout is present) the fixture recipe re-running bit for bit."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import ref_shim
from oracle.lpips_oracle import state_shapes, synthetic_lpips_state
from vidtok_b200 import _native as N
from vidtok_b200 import metrics

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_key_table_matches_the_library_and_the_oracle():
    h = C.c_void_p()
    N.check(N.lib().vt_lpips_create(0, C.byref(h)))
    try:
        native = {}
        for i in range(N.lib().vt_lpips_num_params(h)):
            name, shape, nd = C.create_string_buffer(128), (C.c_int64 * 4)(), C.c_int32()
            N.check(N.lib().vt_lpips_param_info(h, i, name, 128, shape, C.byref(nd)))
            native[name.value.decode()] = tuple(shape[:nd.value])
    finally:
        N.lib().vt_lpips_destroy(h)
    assert native == metrics.lpips_state_shapes() == state_shapes()
    assert len(native) == 31 and native["net.slice5.28.weight"] == (512, 512, 3, 3) and native["lin0.model.1.weight"] == (1, 64, 1, 1)


def test_loader_takes_both_checkpoint_forms_and_refuses_bad_ones():
    ref = synthetic_lpips_state(1)
    ref_full = dict(ref, **{"scaling_layer.shift": torch.tensor([-.030, -.088, -.188])[None, :, None, None],
                            "scaling_layer.scale": torch.tensor([.458, .448, .450])[None, :, None, None]})
    tv = {("features." + k.split(".", 2)[2] if k.startswith("net.") else k): v for k, v in ref.items()}
    tv["classifier.0.weight"] = torch.zeros(4, 4)
    for sd in (ref, ref_full, tv):
        got = metrics.lpips_state(sd)
        assert got.keys() == ref.keys() and all(torch.equal(got[k], ref[k]) for k in ref)
    with pytest.raises(KeyError, match=r"net.slice3.12.weight \(or features.12.weight\)"):
        metrics.lpips_state({k: v for k, v in tv.items() if k != "features.12.weight"})
    with pytest.raises(KeyError, match="lin4.model.1.weight"):
        metrics.lpips_state({k: v for k, v in ref.items() if k != "lin4.model.1.weight"})
    with pytest.raises(ValueError, match=r"net.slice1.2.bias: shape \(63,\)"):
        metrics.lpips_state(dict(ref, **{"net.slice1.2.bias": torch.zeros(63)}))
    with pytest.raises(ValueError, match="scaling_layer.scale"):
        metrics.lpips_state(dict(ref_full, **{"scaling_layer.scale": torch.ones(1, 3, 1, 1)}))
    with pytest.raises(ValueError, match="precision"):
        metrics.LPIPS(ref, precision="fp8")


def test_from_files_never_downloads(tmp_path):
    missing = str(tmp_path / "nowhere" / "vgg16-397923af.pth")
    with pytest.raises(FileNotFoundError, match="nowhere"):
        metrics.LPIPS.from_files(missing, str(tmp_path / "vgg.pth"))
    assert metrics.torchvision_vgg16_path().endswith(os.path.join("hub", "checkpoints", "vgg16-397923af.pth"))


def test_pass_size_rule():
    for H, W in ((256, 256), (16, 16), (480, 640), (1080, 1920), (2160, 3840), (720, 1280)):
        g = metrics.lpips_pass_frames(H, W)
        per = 2 * H * W * 64
        assert 1 <= g <= 16 and g * per <= 2 ** 31 and (g == 16 or (g + 1) * per > 2 ** 31), (H, W, g)
    assert metrics.lpips_pass_frames(256, 256) == 16
    assert metrics.lpips_pass_frames(1080, 1920) == 8       # 16 pairs would be 4.2e9 elements of relu1_2
    assert metrics.lpips_pass_frames(2160, 3840) == 2
    assert metrics.lpips_pass_frames(8192, 8192) == 0


def _ws(h, prec, B, T, H, W):
    return N.lib().vt_lpips_workspace_bytes(h, prec, B, 3, T, H, W)


def test_workspace_without_a_gpu():
    h = C.c_void_p()
    N.check(N.lib().vt_lpips_create(0, C.byref(h)))
    try:
        def expect(esz, B, T, H, W):
            g = min(B * T, metrics.lpips_pass_frames(H, W))
            up = lambda n: (n + 1023) // 1024 * 1024
            tiles, h_, w_ = 0, H, W
            for _ in range(5):
                tiles += (h_ * w_ + 63) // 64
                h_, w_ = h_ // 2, w_ // 2
            return 2 * up(2 * g * H * W * 64 * esz) + up(g * tiles * 4)
        for B, T, H, W in ((8, 17, 256, 256), (1, 17, 1080, 1920), (1, 1, 16, 16), (1, 4, 240, 360), (3, 1, 2160, 3840)):
            assert _ws(h, N.PREC_BF16, B, T, H, W) == expect(2, B, T, H, W)
            assert _ws(h, N.PREC_EXACT_TC, B, T, H, W) == expect(4, B, T, H, W)
        # 8 pairs of 1080p relu1_2 in split rows: beyond 2^32 bytes per buffer
        assert _ws(h, N.PREC_EXACT_TC, 1, 17, 1080, 1920) > 2 * 2 ** 32
        for bad in ((N.PREC_FMA32, 1, 1, 64, 64), (N.PREC_MIXED, 1, 1, 64, 64), (N.PREC_BF16, 1, 1, 15, 64),
                    (N.PREC_BF16, 1, 1, 64, 8), (N.PREC_BF16, 0, 1, 64, 64)):
            assert _ws(h, *bad) == -1
        assert N.lib().vt_lpips_workspace_bytes(h, N.PREC_BF16, 1, 4, 1, 64, 64) == -1
        assert b"C == 3" in N.lib().vt_last_error()
    finally:
        N.lib().vt_lpips_destroy(h)


def test_argument_errors_launch_nothing():
    lib = N.lib()
    h = C.c_void_p()
    N.check(lib.vt_lpips_create(0, C.byref(h)))
    fake = C.c_void_p(0x1000)
    try:
        need = _ws(h, N.PREC_BF16, 1, 2, 64, 64)

        def call(prec=N.PREC_BF16, dt=0, C_=3, H=64, W=64, nbytes=need):
            lib.vt_launch_count(1)
            rc = lib.vt_lpips(h, prec, fake, dt, fake, 0, 1, C_, 2, H, W, fake, None, None, fake, nbytes, None)
            assert lib.vt_launch_count(0) == 0
            return rc

        assert call(prec=N.PREC_FMA32) == -1 and b"BF16 or EXACT_TC" in lib.vt_last_error()
        assert call(dt=3) == -1
        assert call(C_=1) == -1
        assert call(H=8) == -1 and b"16 x 16" in lib.vt_last_error()
        assert call(nbytes=need - 1) == -4
        assert call() == -3                  # arguments fine, parameters never loaded
        assert lib.vt_lpips(h, N.PREC_BF16, None, 0, fake, 0, 1, 3, 2, 64, 64, fake, None, None, fake, need, None) == -1
    finally:
        lib.vt_lpips_destroy(h)


def test_grouping_identity():
    """scripts/inference_evaluate.py appends each group's .mean() once per frame of the group: the mean of that list is the
    mean over frames of the per-frame values, for any grouping, which is what Scorer keeps."""
    rng = np.random.default_rng(0)
    for n in (1, 15, 16, 17, 33, 136):
        v = rng.random(n)
        lst = []
        for i in range(0, n, 16):
            lst += [v[i:i + 16].mean()] * len(v[i:i + 16])
        assert abs(np.mean(lst) - v.mean()) <= 1e-15


@pytest.mark.skipif(not ref_shim.reference_available(), reason="needs the reference checkout")
def test_fixture_recipe_regenerates_bit_identically(tmp_path):
    pytest.importorskip("torchvision")
    env = dict(os.environ, VIDTOK_GOLDEN_LPIPS_OUT=str(tmp_path))
    subprocess.run([sys.executable, os.path.join(ROOT, "oracle", "make_golden_lpips.py")], check=True, env=env, cwd=ROOT,
                   capture_output=True)
    for name in ("lpips_64x64.npz", "lpips_48x80.npz"):
        a, b = np.load(tmp_path / name), np.load(os.path.join(ROOT, "tests", "golden", "lpips", name))
        assert sorted(a.files) == sorted(b.files)
        for k in a.files:
            assert a[k].tobytes() == b[k].tobytes(), (name, k)
