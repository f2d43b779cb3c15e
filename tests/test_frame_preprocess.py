"""ImagePreprocessor (composite on white, crop to the foreground box, pad to a square) — SURVEY 8(f) rank 3, second half.

CPU: the numpy restatement (oracle/preprocess_oracle.py) against the output of the reference's OWN
`ImagePreprocessor.process_images` (actionmesh/preprocessing/image_processor.py) on the frames below, stored by
oracle/gen_golden.py in tests/golden/live_reference.pt.
GPU (-m gpu): B200FramePreprocessor's uint8 output `array_equal` to the restatement, shared and independent cropping,
non-square frames, the invalid-alpha error."""
import numpy as np
import pytest

from conftest import load_golden
from oracle import preprocess_oracle


def _frames(n=5, H=96, W=128, seed=3):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        img = rng.integers(0, 256, (H, W, 4), dtype=np.uint8)
        yy, xx = np.mgrid[0:H, 0:W]
        cy, cx, r = H // 2 + 3 * i - 4, W // 2 - 2 * i, 20 + 2 * i
        d = np.sqrt((yy - cy) ** 2 + (xx - cx) ** 2)
        alpha = np.clip((r + 6 - d) * 40, 0, 255).astype(np.uint8)       # a disc with a soft (partially transparent) edge
        img[..., 3] = alpha
        out.append(img)
    return out


@pytest.mark.parametrize("independent", [False, True])
def test_restatement_matches_the_reference_module(independent):
    ref = load_golden("live_reference.pt")["frame_preprocess"][independent]
    frames = _frames()
    ours = preprocess_oracle.frame_preprocess(frames, independent, 0.1)
    assert len(ref) == len(ours)
    for a, b in zip(ref, ours):
        assert np.array_equal(np.asarray(a), b)
    bad = frames[0].copy()
    bad[..., 3] = 255
    with pytest.raises(ValueError):
        preprocess_oracle.frame_preprocess([bad])


@pytest.mark.gpu
@pytest.mark.parametrize("independent", [False, True])
def test_gpu_frame_preprocessing_is_bit_exact(amb_lib, independent):
    from PIL import Image

    from actionmesh_b200.preprocess import B200FramePreprocessor

    for H, W in ((96, 128), (130, 70)):
        frames = _frames(H=H, W=W, seed=H)
        want = preprocess_oracle.frame_preprocess(frames, independent, 0.1)
        proc = B200FramePreprocessor(independent_cropping=independent, padding_ratio=0.1)
        got = proc.process_images([Image.fromarray(f, "RGBA") for f in frames])
        assert len(got) == len(want)
        for a, b in zip(got, want):
            assert np.array_equal(np.asarray(a), b)
    bad = _frames(n=1)[0]
    bad[..., 3] = 255
    with pytest.raises(ValueError):
        B200FramePreprocessor().process_images([Image.fromarray(bad, "RGBA")])
