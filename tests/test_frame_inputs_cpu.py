"""The resize plan of B200ImagePreprocessor at the sizes a video produces, checked without a GPU.

`_plan` holds everything the two resize kernels are given: the cropped horizontal and vertical coefficient tables and the
window of source rows [y0, y0 + n_rows) the horizontal pass covers.  Driving that plan through a numpy integer convolution
that does what the kernels do (csrc/preprocess.cu) must reproduce Pillow's resize + centre crop bit for bit, for both
DinoV2 settings the pipeline uses: (shortest edge 256, crop 224) for the frame encoder and (518, 518) for TripoSG's.  The
sizes are the frame preprocessor's square-padded crops (near-square both ways, upscales, an exact 2x), single-axis
identity passes and whole 1080p frames."""
import numpy as np
import pytest
import torch
from PIL import Image

from actionmesh_b200.preprocess import PRECISION_BITS, B200ImagePreprocessor
from oracle import preprocess_oracle as po

SETTINGS = [(256, 224), (518, 518)]
SIZES = [(1300, 1299), (1299, 1300), (2303, 2304), (1036, 1036), (300, 300), (98, 97), (600, 518), (518, 700),
         (1080, 1920), (1920, 1080), (256, 300), (518, 518), (1037, 1036)]          # (H, W)


def _plan_on_host(short, crop, H, W):
    p = B200ImagePreprocessor(short, (crop, crop))._plan(H, W, torch.device("cpu"))
    return {k: (v.numpy() if isinstance(v, torch.Tensor) else v) for k, v in p.items()}


def _run_plan(img, plan):
    """The two kernels' integer arithmetic on the host: horizontal pass over the source rows [y0, y0 + n_rows), uint8 between
    the passes, vertical pass indexed relative to y0."""
    y0, n_rows = plan["y0"], plan["n_rows"]
    half = 1 << (PRECISION_BITS - 1)

    def conv(src, bounds, coeffs, axis):
        x = np.moveaxis(src, axis, 0).astype(np.int64)
        acc = np.full((len(bounds),) + x.shape[1:], half, dtype=np.int64)
        for t in range(coeffs.shape[1]):                      # tap t of every output, zero past its tap count
            idx = np.minimum(bounds[:, 0] + t, x.shape[0] - 1)
            w = np.where(t < bounds[:, 1], coeffs[:, t], 0).astype(np.int64)
            acc += x[idx] * w[:, None, None]
        return np.moveaxis(np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8), 0, axis)

    mid = conv(img[y0:y0 + n_rows, :, :3], plan["bh"], plan["kh"], 1)
    bv = plan["bv"].copy()
    bv[:, 0] -= y0
    return conv(mid, bv, plan["kv"], 0)


@pytest.mark.parametrize("short,crop", SETTINGS)
@pytest.mark.parametrize("H,W", SIZES)
def test_resize_plan_reproduces_pillow(short, crop, H, W):
    plan = _plan_on_host(short, crop, H, W)
    assert plan["n_rows"] <= H and plan["bv"][:, 0].min() == plan["y0"]
    rng = np.random.default_rng(H * 7919 + W + short)
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    ref_pv, ref_u8 = po.bit_preprocess_pil([Image.fromarray(img, "RGB")], shortest_edge=short, crop=(crop, crop),
                                           return_u8=True)
    got = _run_plan(img, plan)
    assert np.array_equal(got, ref_u8[0])
    p = B200ImagePreprocessor(short, (crop, crop))
    pv = (p._lut_host[got] - np.array(p.image_mean, dtype=np.float32)) / np.array(p.image_std, dtype=np.float32)
    assert np.array_equal(np.transpose(pv, (2, 0, 1)), ref_pv[0])
