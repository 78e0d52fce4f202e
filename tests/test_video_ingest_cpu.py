"""The output geometry of vidtok_b200.video_io.transform_frames (resized size and centre-crop offset) against torchvision's
Resize(int, antialias=True) + CenterCrop on the CPU, over a grid of source shapes and targets.  No GPU needed."""
import pytest
import torch

from vidtok_b200.video_io import resize_crop_geometry

SOURCES = [(1080, 1920), (1920, 1080), (720, 1280), (240, 320), (256, 340), (2160, 3840), (1081, 1917), (577, 1025),
           (100, 100), (333, 500), (500, 333), (17, 999)]
TARGETS = [(256, 256), (128, 128), (200, 136), (96, 160), (17, 17), (64, 300)]


@pytest.mark.parametrize("src", SOURCES, ids=[f"{h}x{w}" for h, w in SOURCES])
def test_resize_and_crop_geometry_matches_torchvision(src):
    from torchvision import transforms
    Hs, Ws = src
    for H, W in TARGETS:
        resized = transforms.Resize(H, antialias=True)(torch.zeros((1, Hs, Ws)))
        Hr, Wr = resized.shape[1:]
        if H > Hr or W > Wr:                           # torchvision would pad; transform_frames refuses
            with pytest.raises(ValueError, match="crop larger"):
                resize_crop_geometry(Hs, Ws, H, W)
            continue
        # the crop's top-left corner, read back from CenterCrop applied to a position-coded image
        pos = torch.arange(Hr * Wr, dtype=torch.float64).reshape(1, Hr, Wr)
        corner = int(transforms.CenterCrop((H, W))(pos)[0, 0, 0])
        assert resize_crop_geometry(Hs, Ws, H, W) == (Hr, Wr) + divmod(corner, Wr), (src, H, W)
