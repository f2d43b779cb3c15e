"""`actionmesh_b200.video_input.load_frames`: videos, glob patterns and directories, against OpenCV's and PIL's own reads
and the reference's ordering and error rules."""
import numpy as np
import pytest
import torch
from PIL import Image

from actionmesh_b200.video_input import load_frames, natural_sorted


def _rgb(i, h=48, w=64):
    rng = np.random.default_rng(i)
    return rng.integers(0, 255, (h, w, 3), dtype=np.uint8)


def _write_video(path, n):
    import cv2

    h, w = 48, 64
    writer = cv2.VideoWriter(str(path), cv2.VideoWriter_fourcc(*"mp4v"), 8, (w, h))
    yy, xx = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    for k in range(n):
        writer.write(np.stack([(xx * 4 + 6 * k) % 256, yy * 5 % 256, np.full_like(xx, 6 * k)], -1).astype(np.uint8))
    writer.release()


def _opencv_frames(path):
    import cv2

    cap, out = cv2.VideoCapture(str(path)), []
    while True:
        ok, fr = cap.read()
        if not ok:
            break
        out.append(cv2.cvtColor(fr, cv2.COLOR_BGR2RGBA))
    cap.release()
    return out


def _check_timesteps(inp, n):
    assert inp.timesteps.dtype == torch.float32 and torch.equal(inp.timesteps, torch.arange(n, dtype=torch.float32))


@pytest.mark.parametrize("stride,max_frames,n", [(1, None, 40), (1, 31, 31), (2, None, 20), (2, 16, 16)])
def test_video(tmp_path, stride, max_frames, n):
    path = tmp_path / "clip.mp4"
    _write_video(path, 40)
    decoded = _opencv_frames(path)
    assert len(decoded) == 40
    inp = load_frames(path, max_frames=max_frames, stride=stride)
    assert inp.n_frames == n
    _check_timesteps(inp, n)
    for got, want in zip(inp.frames, decoded[::stride][:n]):
        assert isinstance(got, Image.Image) and got.mode == "RGBA" and np.array_equal(np.asarray(got), want)


def test_video_stride_3_and_cap(tmp_path):
    path = tmp_path / "clip.mp4"
    _write_video(path, 40)
    with pytest.raises(AssertionError, match="At least 16 frames are required, got 14"):
        load_frames(path, stride=3)
    _write_video(path, 60)
    inp = load_frames(path, max_frames=31, stride=3)
    assert inp.n_frames == 20
    decoded = _opencv_frames(path)
    assert all(np.array_equal(np.asarray(a), b) for a, b in zip(inp.frames, decoded[::3]))


def test_directory_natural_order_and_glob(tmp_path):
    for i in range(1, 21):
        Image.fromarray(_rgb(i)).save(tmp_path / f"f{i}.png")
    for inp in (load_frames(tmp_path), load_frames(tmp_path / "f*.png")):
        assert inp.n_frames == 20
        _check_timesteps(inp, 20)
        for i, fr in enumerate(inp.frames, start=1):         # f1, f2, ..., f10, not f1, f10, f11, ...
            assert fr.mode == "RGBA" and np.array_equal(np.asarray(fr)[..., :3], _rgb(i))
    with pytest.raises(AssertionError, match="got 9"):         # f?.png: f1 ... f9 only
        load_frames(tmp_path / "f?.png")
    assert [p.name for p in natural_sorted(tmp_path.glob("f1*.png"))][:3] == ["f1.png", "f10.png", "f11.png"]


def test_directory_stride_then_max_frames(tmp_path):
    for i in range(40):
        Image.fromarray(_rgb(i)).save(tmp_path / f"img_{i}.png")
    inp = load_frames(tmp_path, stride=2, max_frames=17)
    assert inp.n_frames == 17
    assert all(np.array_equal(np.asarray(fr)[..., :3], _rgb(2 * k)) for k, fr in enumerate(inp.frames))


def test_image_mask_pairs(tmp_path):
    masks = {}
    for i in range(16):
        Image.fromarray(_rgb(i)).save(tmp_path / f"{i:03d}_image.png")
        size = (32, 24) if i % 2 else (64, 48)                    # every other mask at a different size
        mask = Image.fromarray(np.random.default_rng(100 + i).integers(0, 255, size[::-1], dtype=np.uint8), "L")
        mask.save(tmp_path / f"{i:03d}_mask.png")
        masks[i] = mask if mask.size == (64, 48) else mask.resize((64, 48), Image.LANCZOS)
    Image.fromarray(_rgb(99)).save(tmp_path / "zzz.jpg")           # ignored: pairs take precedence
    inp = load_frames(tmp_path)
    assert inp.n_frames == 16
    for i, fr in enumerate(inp.frames):
        arr = np.asarray(fr)
        assert fr.mode == "RGBA" and np.array_equal(arr[..., :3], _rgb(i)) and np.array_equal(arr[..., 3], masks[i])
    (tmp_path / "003_mask.png").rename(tmp_path / "003_other.png")
    with pytest.raises(ValueError, match="No mask found for 003_image.png"):
        load_frames(tmp_path)


def test_png_is_preferred_over_jpg(tmp_path):
    for i in range(16):
        Image.fromarray(_rgb(i)).save(tmp_path / f"a{i}.png")
    for i in range(20):
        Image.fromarray(_rgb(50 + i)).save(tmp_path / f"b{i}.jpg")
    inp = load_frames(tmp_path)
    assert inp.n_frames == 16 and np.array_equal(np.asarray(inp.frames[5])[..., :3], _rgb(5))
    jpg_only = tmp_path / "jpg"
    jpg_only.mkdir()
    for i in range(16):
        Image.fromarray(_rgb(i)).save(jpg_only / f"{i}.jpeg")
    assert load_frames(jpg_only).n_frames == 16


def test_errors(tmp_path):
    for i in range(15):
        Image.fromarray(_rgb(i)).save(tmp_path / f"{i}.png")
    with pytest.raises(AssertionError, match="At least 16 frames are required, got 15"):
        load_frames(tmp_path)
    with pytest.raises(FileNotFoundError, match="Video file not found"):
        load_frames(tmp_path / "missing.mp4")
    (tmp_path / "broken.mp4").write_bytes(b"not a video")
    with pytest.raises(RuntimeError, match="Failed to open video"):
        load_frames(tmp_path / "broken.mp4")
    with pytest.raises(ValueError, match="Unsupported input"):
        load_frames(tmp_path / "0.png")
    (tmp_path / "empty").mkdir()
    with pytest.raises(ValueError, match="No images found in directory"):
        load_frames(tmp_path / "empty")
    with pytest.raises(ValueError, match="No images found matching"):
        load_frames(tmp_path / "*.webp")
