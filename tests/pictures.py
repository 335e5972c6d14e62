"""The pictures the DINOv2 tests feed: the fixture picture of tests/golden/dinov2.npz (tests/golden/make_golden.py builds it the same
way, and tests/test_ref_modules_host.py pins it to the fixture through the reference module), its 224 x 224 crop, and the same picture
as inference.py builds its input.  numpy only."""
import numpy as np


def golden_picture(seed):
    """The 518 x 518 picture of dinov2.npz (a smooth colour field + noise, 0..255), [1, 518, 518, 3] fp32 numpy."""
    rs = np.random.RandomState(seed)
    yy, xx = np.meshgrid(np.linspace(0, 1, 518), np.linspace(0, 1, 518), indexing="ij")
    img = np.stack([127 + 100 * np.sin(6 * xx + 2 * yy), 127 + 100 * np.cos(5 * yy), 255 * xx * yy], -1) + 12 * rs.standard_normal((518, 518, 3))
    return np.clip(img, 0, 255).astype(np.float32)[None]


def small_picture(img):
    """The fixture's 224 x 224 picture (every second pixel of the 518 x 518 one): it goes through Resize(518, bicubic)."""
    return np.ascontiguousarray(np.clip(img[:, ::2, ::2][:, :224, :224], 0, 255))


def masked_picture(img):
    """inference.py:306-311 on the fixture picture: a uint8 RGB picture times the int64 mask (alpha > 0) * 1 of a centred disc -> int64
    [1, 518, 518, 3], background zero."""
    yy, xx = np.mgrid[:518, :518]
    alpha = np.where((yy - 258.5) ** 2 + (xx - 258.5) ** 2 <= 215 ** 2, 255, 0).astype(np.uint8)
    mask = (alpha[..., None] > 0) * 1
    out = img[0].astype(np.uint8) * mask
    assert out.dtype == np.int64
    return out[None]
