"""Frame cropping and DinoV2 preprocessing on the GPU at the sizes a video produces (-m gpu), bit for bit against numpy and
Pillow.

- `ops.alpha_stats` against numpy at widths on both sides of one CTA (256 px), of the four-CTA row split and of its strided
  loop (1024 px), up to 4K, at heights 1 to 2160, with a different alpha pattern in each of up to 16 frames per call.
- `ops.composite_crop_pad` on every (colour byte, alpha byte) pair, then on crop boxes touching each frame edge, a 1x1 box and
  zero and asymmetric paddings of 16 1080p frames.
- The resize kernels against Pillow for 16 frames at each size the frame preprocessor emits, at both DinoV2 settings:
  (shortest edge 256, crop 224) for the frame encoder and (518, 518) for TripoSG's.  The pipeline's 16 frames already run
  more outputs than one grid of the vertical kernel covers (16 CTAs of 256 threads per SM).
- The whole chain: B200FramePreprocessor on 16 soft-masked 1080p frames, then both DinoV2 preprocessors, against
  preprocess_oracle.frame_preprocess and Pillow; and the foreground-ratio check at its exact boundary."""
import numpy as np
import pytest
import torch
from PIL import Image

from oracle import preprocess_oracle as po

pytestmark = pytest.mark.gpu

WIDTHS = [1, 31, 255, 256, 257, 1023, 1024, 1025, 1920, 3840, 4097]
HEIGHTS = [1, 7, 1080, 2160]


def _alpha_patterns(H, W, rng):
    """One (H, W) uint8 alpha plane per pattern."""
    yy, xx = np.mgrid[0:H, 0:W]
    out = [np.zeros((H, W), np.uint8)]                                      # nothing: the sentinels
    a = np.zeros((H, W), np.uint8)
    a[0, 0], a[0, W - 1], a[H - 1, 0], a[H - 1, W - 1] = 1, 200, 128, 127   # one pixel at each corner
    out.append(a)
    for sl in ((slice(None), 0), (slice(None), W - 1), (0, slice(None)), (H - 1, slice(None))):
        a = np.zeros((H, W), np.uint8)                                      # first / last column, first / last row only
        a[sl] = rng.integers(1, 256, a[sl].shape)
        out.append(a)
    out.append(np.choose((xx + 2 * yy) % 3, [0, 127, 128]).astype(np.uint8))  # 127 against 128 at the > 127 count
    out.append(np.full((H, W), 255, np.uint8))
    a = np.zeros((H, W), np.uint8)                                          # one pixel somewhere inside
    a[rng.integers(H), rng.integers(W)] = 130
    out.append(a)
    out.append((rng.integers(0, 256, (H, W)) * (rng.random((H, W)) < 0.001)).astype(np.uint8))  # sparse random
    out.append(rng.integers(0, 256, (H, W), dtype=np.uint8))                # dense random
    return out


def _alpha_stats_numpy(a):
    H, W = a.shape
    m = a > 0
    rows, cols = np.flatnonzero(m.any(1)), np.flatnonzero(m.any(0))
    box = [cols[0], rows[0], cols[-1], rows[-1]] if len(rows) else [W, H, -1, -1]
    return box + [int(np.count_nonzero(a > 127))]


@pytest.mark.parametrize("H", HEIGHTS)
@pytest.mark.parametrize("W", WIDTHS)
def test_alpha_stats_matches_numpy(amb_lib, H, W):
    from actionmesh_b200 import ops

    rng = np.random.default_rng(H * 10007 + W)
    alphas = _alpha_patterns(H, W, rng)
    assert len(alphas) <= 16
    rgba = np.zeros((len(alphas), H, W, 4), np.uint8)
    rgba[..., 3] = np.stack(alphas)
    rgba[..., :3] = 255                                                       # colour must not leak into the stats
    got = ops.alpha_stats(torch.from_numpy(rgba).cuda()).cpu().numpy()
    want = np.array([_alpha_stats_numpy(a) for a in alphas])
    assert np.array_equal(got, want), (H, W, np.flatnonzero((got != want).any(1)))


def _composite_numpy(rgba, box, px, py):
    """preprocess_oracle.frame_preprocess's composite, crop, pad and uint8 conversion for a given box and padding, in its
    float32 operation order."""
    bg = np.array([1.0, 1.0, 1.0]).astype(np.float32)
    x, y, w, h = box
    out = []
    for img in rgba:
        rgb, alpha = img[..., :3], img[..., 3]
        a = (alpha.astype(np.float32) * (1.0 / 255.0))[..., None]
        comp = rgb.astype(np.float32) * (1.0 / 255.0) * a + bg * (1.0 - a)
        padded = np.pad(comp[y:y + h, x:x + w], ((py, py), (px, px), (0, 0)), mode="constant", constant_values=1.0)
        out.append((padded * np.float32(255)).astype(np.uint8))
    return np.stack(out)


def _every_pair_frames():
    """Two 256x256 frames in which each (colour byte, alpha byte) pair occurs in every channel: pixel (row a, column v) has
    colour bytes (v, 91 v + 17 mod 256, 255 - v).  The second frame's alpha is shifted by one row, so that the union of the
    two foreground boxes is the whole frame and the crop keeps the alpha-0 row."""
    v = np.arange(256)
    rgb = np.stack([v, (91 * v + 17) % 256, 255 - v], -1).astype(np.uint8)
    frames = np.empty((2, 256, 256, 4), np.uint8)
    frames[:, :, :, :3] = rgb[None, None]
    frames[0, :, :, 3] = v[:, None]
    frames[1, :, :, 3] = ((v + 1) % 256)[:, None]
    return frames


def test_composite_every_value_alpha_pair(amb_lib):
    from actionmesh_b200 import ops

    frames = _every_pair_frames()
    want = po.frame_preprocess(list(frames), independent_cropping=False, padding_ratio=0.0)
    assert all(w.shape == (256, 256, 3) for w in want)
    assert np.array_equal(_composite_numpy(frames, (0, 0, 256, 256), 0, 0), np.stack(want))
    got = ops.composite_crop_pad(torch.from_numpy(frames).cuda(), (0, 0, 256, 256), 0, 0).cpu().numpy()
    for c in range(3):
        bad = np.argwhere(got[0, :, :, c] != want[0][:, :, c])
        assert not len(bad), f"channel {c}: {len(bad)} (alpha, column) pairs differ, first {bad[:4].tolist()}"
    assert np.array_equal(got[1], want[1])


@pytest.mark.parametrize("H,W", [(1080, 1920), (1920, 1080)])
def test_composite_boxes_at_the_frame_edges(amb_lib, H, W):
    from actionmesh_b200 import ops

    rng = np.random.default_rng(H)
    frames = rng.integers(0, 256, (16, H, W, 4), dtype=np.uint8)
    frames[:, :, :, 3][rng.random((16, H, W)) < 0.2] = 0
    frames[:, :, :, 3][rng.random((16, H, W)) < 0.2] = 255
    dev = torch.from_numpy(frames).cuda()
    cases = [((0, 100, 300, 200), 0, 0), ((W - 300, 50, 300, 400), 3, 17), ((500, 0, 200, 100), 40, 0),
             ((60, H - 150, 250, 150), 0, 25), ((0, 0, 1, 1), 0, 0), ((W - 1, H - 1, 1, 1), 5, 2), ((0, 0, W, H), 0, 0),
             ((0, 0, W, H), 7, 1), ((W - 1, 0, 1, H), 3, 0), ((0, H - 1, W, 1), 0, 4)]
    for box, px, py in cases:
        got = ops.composite_crop_pad(dev, box, px, py).cpu().numpy()
        want = _composite_numpy(frames, box, px, py)
        assert got.shape == want.shape and np.array_equal(got, want), (box, px, py)


RESIZE_SIZES = [(1300, 1299), (1299, 1300), (2303, 2304), (1036, 1036), (300, 300), (98, 97), (600, 518), (518, 700),
                (1080, 1920), (1920, 1080)]                                     # (H, W)


@pytest.mark.parametrize("short,crop", [(256, 224), (518, 518)])
@pytest.mark.parametrize("k", range(len(RESIZE_SIZES)))
def test_resize_16_frames_matches_pillow(amb_lib, short, crop, k):
    from actionmesh_b200.preprocess import B200ImagePreprocessor

    H, W = RESIZE_SIZES[k]
    mode = "RGBA" if (k + (short == 518)) % 2 else "RGB"                      # every size in both modes over the two settings
    rng = np.random.default_rng(k * 31 + short)
    frames = rng.integers(0, 256, (16, H, W, len(mode)), dtype=np.uint8)
    ref_pv, ref_u8 = po.bit_preprocess_pil([Image.fromarray(f, mode) for f in frames], shortest_edge=short,
                                           crop=(crop, crop), return_u8=True)
    pv, u8 = B200ImagePreprocessor(short, (crop, crop)).preprocess_u8(torch.from_numpy(frames), "cuda", return_u8=True)
    assert np.array_equal(u8.cpu().numpy(), ref_u8)
    assert np.array_equal(pv.cpu().numpy().view(np.uint32), ref_pv.view(np.uint32))


def _soft_masked_frames(H, W, seed):
    """16 RGBA frames with soft-edged discs: frames 0-3 reach past one frame edge each, the others lie inside."""
    rng = np.random.default_rng(seed)
    frames = rng.integers(0, 256, (16, H, W, 4), dtype=np.uint8)
    yy, xx = np.mgrid[0:H, 0:W]
    s = min(H, W)
    for i in range(16):
        r = s * (0.15 + 0.01 * i)
        cy, cx = H / 2 + rng.uniform(-0.15, 0.15) * s, W / 2 + rng.uniform(-0.15, 0.15) * s
        if i < 4:
            cy, cx = ((-0.1 * s, cx), (H + 0.1 * s, cx), (cy, -0.1 * s), (cy, W + 0.1 * s))[i]
            r = 0.3 * s
        d = np.sqrt((yy - cy) ** 2 + (xx - cx) ** 2)
        frames[i, :, :, 3] = np.clip((r + 6 - d) * 40, 0, 255).astype(np.uint8)
    return frames


@pytest.fixture(scope="module")
def masked_frames():
    return {(H, W): _soft_masked_frames(H, W, H) for H, W in ((1080, 1920), (1920, 1080))}


@pytest.mark.parametrize("ratio", [0.0, 0.1, 0.5])
@pytest.mark.parametrize("independent", [False, True])
@pytest.mark.parametrize("H,W", [(1080, 1920), (1920, 1080)])
def test_full_chain_matches_oracle_and_pillow(amb_lib, masked_frames, H, W, independent, ratio):
    from actionmesh_b200.preprocess import B200FramePreprocessor, B200ImagePreprocessor

    frames = masked_frames[(H, W)]
    want = po.frame_preprocess(list(frames), independent_cropping=independent, padding_ratio=ratio)
    got = B200FramePreprocessor(independent_cropping=independent, padding_ratio=ratio).process_to_u8(
        [Image.fromarray(f, "RGBA") for f in frames])
    assert len(got) == len(want) == 16
    for g, w in zip(got, want):
        assert tuple(g.shape) == w.shape and np.array_equal(g.cpu().numpy(), w)
    for short, crop in ((256, 224), (518, 518)):
        proc = B200ImagePreprocessor(short, (crop, crop))
        ref_pv, ref_u8 = po.bit_preprocess_pil([Image.fromarray(w, "RGB") for w in want], shortest_edge=short,
                                               crop=(crop, crop), return_u8=True)
        if independent:
            outs = [proc.preprocess_u8(g[None], "cuda", return_u8=True) for g in got]
            pv, u8 = torch.cat([o[0] for o in outs]), torch.cat([o[1] for o in outs])
        else:
            pv, u8 = proc.preprocess_u8(torch.stack(got), "cuda", return_u8=True)
        assert np.array_equal(u8.cpu().numpy(), ref_u8)
        assert np.array_equal(pv.cpu().numpy().view(np.uint32), ref_pv.view(np.uint32))


@pytest.mark.parametrize("H,W", [(1080, 1920), (97, 131)])
def test_foreground_ratio_boundary(amb_lib, H, W):
    from actionmesh_b200.preprocess import B200FramePreprocessor

    min_count = int(H * W * 0.01)
    rng = np.random.default_rng(W)
    base = rng.integers(0, 256, (H, W, 4), dtype=np.uint8)

    def frame(fg, soft=0):
        """`fg` pixels of alpha 255 then `soft` pixels of alpha 127 (inside the box, not counted), the rest alpha 0."""
        f = base.copy()
        a = np.zeros(H * W, np.uint8)
        a[:fg] = 255
        a[fg:fg + soft] = 127
        f[..., 3] = a.reshape(H, W)
        return f

    proc = B200FramePreprocessor(padding_ratio=0.1)
    for fg, soft in ((min_count, 3), (H * W - min_count, 0)):                # both sides accepted at the boundary
        f = frame(fg, soft)
        got = proc.process_to_u8([Image.fromarray(f, "RGBA")])
        assert np.array_equal(got[0].cpu().numpy(), po.frame_preprocess([f], False, 0.1)[0])
    for fg in (min_count - 1, H * W - min_count + 1):                          # one pixel past it on either side
        with pytest.raises(ValueError):
            po.frame_preprocess([frame(fg)])
        with pytest.raises(ValueError):
            proc.process_to_u8([Image.fromarray(frame(fg), "RGBA")])
