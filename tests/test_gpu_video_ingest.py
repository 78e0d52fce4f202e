"""-m gpu: device ingest of decoded frames (vidtok_b200.video_io.transform_frames) against the reference's transform run with
torchvision on the CPU (vidtok/data/vidtok.py:51-56,181-185; scripts/inference_reconstruct.py:41-47,73-74):

    Resize(input_height, antialias=True) -> CenterCrop((input_height, input_width)) -> Normalize(.5, .5)
    on frames.permute(0, 3, 1, 2).float() / 255, then .permute(1, 0, 2, 3)

The kernel restates torch's CPU antialiased bilinear resize op by op, including the order and rounding of its compiled tap
sum (groups of four taps through an in-order vector reduction, FMA for the rest).  That compiled sum belongs to one CPU
build of torch: on the AVX512 kernels of the x86 wheel every case is bit-identical, and that is asserted there.  Elsewhere
the bound is 4.8e-7 on the normalised clip (4 ulp just above 1.0; the sum order is the same, only the contraction of the
last taps may differ).
"""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

from vidtok_b200 import _native as N  # noqa: E402
from vidtok_b200.video_io import resize_crop_geometry, transform_frames  # noqa: E402

TOL = 4.8e-7
BIT_EXACT = torch.backends.cpu.get_cpu_capability() == "AVX512"


def reference(frames, H, W):
    from torchvision import transforms
    Cc = frames.shape[-1]
    tf = transforms.Compose([transforms.Resize(H, antialias=True), transforms.CenterCrop((H, W)),
                             transforms.Normalize(mean=(0.5,) * Cc, std=(0.5,) * Cc)])
    return tf(frames.permute(0, 3, 1, 2).float() / 255.0).permute(1, 0, 2, 3)     # [C,T,H,W]


def frames_for(N_, Hs, Ws, Cc, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (N_, Hs, Ws, Cc), generator=g, dtype=torch.uint8)


def compare(name, got, ref):
    same = float((got == ref).double().mean())
    err = float((got - ref).abs().max())
    print(f"{name}: bit-identical {same:.6f}, max |d| {err:.3g}")
    assert err <= TOL, f"{name}: max |d| {err} > {TOL}"
    if BIT_EXACT:
        assert same == 1.0, f"{name}: only {same:.6f} of the outputs are bit-identical on this CPU build"


# (id, N, Hs, Ws, C, H, W)
CASES = [
    ("mcljcv_1080p_256", 17, 1080, 1920, 3, 256, 256),      # MCL-JCV evaluation protocol
    ("1080p_128", 4, 1080, 1920, 3, 128, 128),              # scripts/inference_reconstruct.py default
    ("720p_256", 4, 720, 1280, 3, 256, 256),
    ("portrait_256", 3, 1920, 1080, 3, 256, 256),
    ("upscale_240p_256", 4, 240, 320, 3, 256, 256),
    ("identity_256", 4, 256, 340, 3, 256, 256),             # short side already 256: the resize returns the frame
    ("4k_128", 2, 2160, 3840, 3, 128, 128),                 # scale ~17: small tiles
    ("odd_1081x1917_200x136", 3, 1081, 1917, 3, 200, 136),
    ("c1_1080p_256", 3, 1080, 1920, 1, 256, 256),
    ("c1_odd_577x1025_96x160", 5, 577, 1025, 1, 96, 160),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_transform_frames_matches_reference(case):
    name, N_, Hs, Ws, Cc, H, W = case
    frames = frames_for(N_, Hs, Ws, Cc, seed=N_ * 1000 + Hs)
    got = transform_frames(frames.cuda(), H, W)
    torch.cuda.synchronize()
    assert tuple(got.shape) == (1, Cc, N_, H, W) and got.dtype == torch.float32
    compare(name, got[0].cpu(), reference(frames, H, W))


def test_transform_frames_splits_clips():
    """34 frames with clip_frames=17 -> [2,3,17,H,W]; each clip equals the reference applied to that clip alone."""
    frames = frames_for(34, 720, 1280, 3, seed=7)
    got = transform_frames(frames.cuda(), 256, 256, clip_frames=17).cpu()
    assert tuple(got.shape) == (2, 3, 17, 256, 256)
    for k in range(2):
        compare(f"clip{k}", got[k], reference(frames[17 * k:17 * (k + 1)], 256, 256))


def test_transform_frames_rejects_bad_input():
    frames = torch.zeros((4, 100, 200, 3), dtype=torch.uint8, device="cuda")
    with pytest.raises(ValueError, match="crop larger"):
        transform_frames(frames, 64, 200)                 # resized to 64x128
    with pytest.raises(ValueError, match="do not split"):
        transform_frames(frames, 64, 64, clip_frames=3)


def test_abi_rejects_crop_outside_resized_frame():
    frames = torch.zeros((2, 100, 200, 3), dtype=torch.uint8, device="cuda")
    clip = torch.empty((1, 3, 2, 64, 64), dtype=torch.float32, device="cuda")
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    f, c = C.c_void_p(frames.data_ptr()), C.c_void_p(clip.data_ptr())
    L = N.lib()
    assert L.vt_video_u8_to_clip_resized(f, c, 2, 100, 200, 3, 64, 128, 1, 0, 64, 64, 2, s) == -1
    assert b"outside the resized frame" in L.vt_last_error()
    assert L.vt_video_u8_to_clip_resized(f, c, 2, 100, 200, 3, 64, 128, 0, 65, 64, 64, 2, s) == -1
    assert L.vt_video_u8_to_clip_resized(f, c, 2, 100, 200, 3, 64, 128, 0, 0, 64, 64, 3, s) == -1     # N % Tc != 0
    assert L.vt_video_u8_to_clip_resized(None, c, 2, 100, 200, 3, 64, 128, 0, 0, 64, 64, 2, s) == -1
    assert L.vt_video_u8_to_clip_resized(f, c, 2, 100, 200, 3, 64, 128, 0, 32, 64, 64, 2, s) == 0
    torch.cuda.synchronize()


def test_scale_beyond_the_smallest_tile_is_an_error():
    """A 1x1 output tile of a ~260x downscale needs a ~530x530x3 byte source window: more than shared memory holds."""
    frames = torch.zeros((1, 4200, 4200, 3), dtype=torch.uint8, device="cuda")
    assert resize_crop_geometry(4200, 4200, 16, 16) == (16, 16, 0, 0)
    with pytest.raises(RuntimeError, match="scale too large"):
        transform_frames(frames, 16, 16)
    # a 110x downscale still fits one 1x1 tile, and runs
    small = frames_for(1, 1100, 1100, 3, seed=3)
    compare("scale_110", transform_frames(small.cuda(), 10, 10)[0].cpu(), reference(small, 10, 10))
