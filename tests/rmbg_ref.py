"""fp32 PyTorch restatement of the reference's background removal, for the tests (CPU, or CUDA with TF32 on or off).

Each function follows the reference line it cites: actionmesh/preprocessing/background_removal.py (pre-processing,
post-processing, refinement, forward) and third_party/TripoSG/scripts/briarmbg.py (BriaRMBG).  OpenCV computes Otsu's
threshold and scipy.ndimage.label with a 3x3 structure labels the components (skimage.measure.label's 2-D default,
connectivity 2).  Also here: seeded synthetic weights with RMS-calibrated BatchNorm statistics, Otsu and bilinear
resampling restated in the kernels' operation order (numpy), and the component filter.
"""
from __future__ import annotations

import functools

import numpy as np
import torch
import torch.nn.functional as F

from actionmesh_b200.background_removal import DECODER, ENCODER, IGNORED_HEADS, conv_layers, rsu_convs

FLT_EPSILON = float(np.finfo(np.float32).eps)
CALIBRATION_SIZE = (256, 320)


# ---- weights ---------------------------------------------------------------------------------------------------------------
def synthetic_frame(h: int, w: int, seed: int) -> np.ndarray:
    """A deterministic (h, w, 3) uint8 frame: a bright blob on a darker gradient, with noise."""
    g = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    blob = np.exp(-(((y - 0.45 * h) / (0.25 * h)) ** 2 + ((x - 0.55 * w) / (0.2 * w)) ** 2))
    base = 60 + 40 * x / max(w - 1, 1)
    img = base[..., None] + 150 * blob[..., None] * np.array([1.0, 0.8, 0.6]) + g.normal(0, 12, (h, w, 3))
    return np.clip(img, 0, 255).astype(np.uint8)


def _conv_init(g: torch.Generator, o: int, i: int):
    """nn.Conv2d's default init: weight and bias U(-1/sqrt(fan_in), 1/sqrt(fan_in))."""
    bound = 1.0 / (9 * i) ** 0.5
    return (torch.rand(o, i, 3, 3, generator=g) * 2 - 1) * bound, (torch.rand(o, generator=g) * 2 - 1) * bound


@functools.lru_cache(maxsize=3)
def make_state_dict(seed: int = 0, calibration_size: tuple = CALIBRATION_SIZE, device: str = "cpu") -> dict:
    """BriaRMBG's full state dict (side2-side6 and num_batches_tracked included): default-init convolutions, BN gamma
    U(0.5, 1.5), beta N(0, 0.1); running statistics calibrated layer by layer in forward order, in fp64 on `device`, on
    synthetic_frame(calibration_size) at that model input size, as RMS statistics (running_mean = 0, running_var = E[x^2]).
    Calibrate at the size a test runs: statistics taken at another size leave a random network that amplifies rounding
    (at 1024 x 1024 with 256 x 320 statistics, TF32 operands move sigmoid(d1) by up to 1.0)."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for prefix, cin, cout, _, bn in conv_layers():
        key = f"{prefix}.conv_s1" if bn else prefix
        sd[f"{key}.weight"], sd[f"{key}.bias"] = _conv_init(g, cout, cin)
        if bn:
            bp = f"{prefix}.bn_s1"
            sd[f"{bp}.weight"] = torch.rand(cout, generator=g) + 0.5
            sd[f"{bp}.bias"] = torch.randn(cout, generator=g) * 0.1
            sd[f"{bp}.running_mean"] = torch.zeros(cout)
            sd[f"{bp}.running_var"] = torch.ones(cout)
            sd[f"{bp}.num_batches_tracked"] = torch.tensor(0)
    for i, c in zip(range(1, 7), (64, 64, 128, 256, 512, 512)):
        sd[f"side{i}.weight"], sd[f"side{i}.bias"] = _conv_init(g, 1, c)
    x = preprocess(synthetic_frame(*calibration_size, seed=1000 + seed), calibration_size, device).double()
    with torch.no_grad():
        rmbg_forward(sd, x, calibrate=True)
    return {k: v.clone() for k, v in sd.items()}


# ---- BriaRMBG (briarmbg.py) ------------------------------------------------------------------------------------------------
def _rebnconv(sd: dict, prefix: str, x: torch.Tensor, dil: int, calibrate: bool) -> torch.Tensor:
    """REBNCONV: conv3x3 (dilation d, padding d) -> BatchNorm (eval, eps 1e-5) -> ReLU (briarmbg.py:13-26)."""
    y = F.conv2d(x, sd[f"{prefix}.conv_s1.weight"].to(x), sd[f"{prefix}.conv_s1.bias"].to(x), padding=dil, dilation=dil)
    bp = f"{prefix}.bn_s1"
    if calibrate:
        sd[f"{bp}.running_var"] = y.double().pow(2).mean((0, 2, 3)).float().cpu()
    y = F.batch_norm(y, sd[f"{bp}.running_mean"].to(x), sd[f"{bp}.running_var"].to(x), sd[f"{bp}.weight"].to(x),
                     sd[f"{bp}.bias"].to(x), False, 0.0, 1e-5)
    return F.relu(y)


def _up(src: torch.Tensor, tar: torch.Tensor) -> torch.Tensor:
    """_upsample_like (briarmbg.py:29-33)."""
    return F.interpolate(src, size=tar.shape[2:], mode="bilinear")


def _pool(x: torch.Tensor) -> torch.Tensor:
    return F.max_pool2d(x, 2, 2, ceil_mode=True)


def _rsu(sd: dict, stage: str, depth: int, x: torch.Tensor, calibrate: bool) -> torch.Tensor:
    """RSU7/6/5/4 (briarmbg.py:74-116, 149-186, 214-244, 268-292) and RSU4F (:312-328)."""
    names = [n for n, *_ in rsu_convs(depth, 1, 1, 1)]
    dil = {n: d for n, _, _, d in rsu_convs(depth, 1, 1, 1)}
    conv = lambda n, t: _rebnconv(sd, f"{stage}.{n}", t, dil[n], calibrate)
    assert names[0] == "rebnconvin"
    hxin = conv("rebnconvin", x)
    if depth == 0:
        hx1 = conv("rebnconv1", hxin)
        hx2 = conv("rebnconv2", hx1)
        hx3 = conv("rebnconv3", hx2)
        hx4 = conv("rebnconv4", hx3)
        hx3d = conv("rebnconv3d", torch.cat((hx4, hx3), 1))
        hx2d = conv("rebnconv2d", torch.cat((hx3d, hx2), 1))
        return conv("rebnconv1d", torch.cat((hx2d, hx1), 1)) + hxin
    enc, h = [], hxin
    for i in range(1, depth):
        enc.append(conv(f"rebnconv{i}", h))
        h = _pool(enc[-1]) if i < depth - 1 else enc[-1]
    d = conv(f"rebnconv{depth}", enc[-1])
    for i in range(depth - 1, 0, -1):
        d = conv(f"rebnconv{i}d", torch.cat((d, enc[i - 1]), 1))
        if i > 1:
            d = _up(d, enc[i - 2])
    return d + hxin


def rmbg_forward(sd: dict, x: torch.Tensor, calibrate: bool = False, return_logits: bool = False):
    """BriaRMBG.forward's result[0][0] = sigmoid(upsample(side1(hx1d), x)) (briarmbg.py:397-463; side2-6 unused)."""
    hx = F.conv2d(x, sd["conv_in.weight"].to(x), sd["conv_in.bias"].to(x), stride=2, padding=1)
    feats = []
    for i, (stage, depth, *_) in enumerate(ENCODER):
        hx = _rsu(sd, stage, depth, hx, calibrate)
        feats.append(hx)
        if i < len(ENCODER) - 1:
            hx = _pool(hx)
    d = feats[-1]
    for j, (stage, depth, *_) in enumerate(DECODER):
        skip = feats[-2 - j]
        d = _rsu(sd, stage, depth, torch.cat((_up(d, skip), skip), 1), calibrate)
    logits = F.conv2d(d, sd["side1.weight"].to(x), sd["side1.bias"].to(x), padding=1)
    soft = torch.sigmoid(_up(logits, x))
    return (soft, logits, d) if return_logits else soft


# ---- background_removal.py -------------------------------------------------------------------------------------------------
def preprocess(im: np.ndarray, size: tuple, device="cpu") -> torch.Tensor:
    """_preprocess_image (background_removal.py:57-69)."""
    t = torch.tensor(im, dtype=torch.float32, device=device).permute(2, 0, 1)
    t = F.interpolate(t[None], size=tuple(size), mode="bilinear", align_corners=False)
    return (t / 255.0 - 0.5) / 1.0


def postprocess_mask(result: torch.Tensor, im_size: tuple) -> np.ndarray:
    """_postprocess_mask (background_removal.py:71-82)."""
    r = torch.squeeze(F.interpolate(result, size=tuple(im_size), mode="bilinear", align_corners=False), 0)
    ma, mi = torch.max(r), torch.min(r)
    r = (r - mi) / (ma - mi)
    return np.squeeze((r * 255).permute(1, 2, 0).cpu().numpy().astype(np.uint8))


def otsu_cv2(mask: np.ndarray) -> tuple[int, np.ndarray]:
    import cv2

    t, binary = cv2.threshold(mask, 0, 255, cv2.THRESH_BINARY + cv2.THRESH_OTSU)
    return int(t), binary


def otsu_threshold(hist) -> int:
    """OpenCV's Otsu threshold of a 256-bin histogram, restated in double precision (DESIGN §17)."""
    h = [int(v) for v in hist]
    n = sum(h)
    scale = 1.0 / n
    mu = sum(i * h[i] for i in range(256)) * scale
    q1 = mu1 = max_sigma = 0.0
    t = 0
    for i in range(256):
        p = h[i] * scale
        mu1 *= q1
        q1 += p
        q2 = 1.0 - q1
        if min(q1, q2) < FLT_EPSILON or max(q1, q2) > 1.0 - FLT_EPSILON:
            continue
        mu1 = (mu1 + i * p) / q1
        mu2 = (mu - q1 * mu1) / q2
        sigma = q1 * q2 * (mu1 - mu2) * (mu1 - mu2)
        if sigma > max_sigma:
            max_sigma, t = sigma, i
    return t


def filter_components(binary: np.ndarray, min_size: int) -> np.ndarray:
    """label (8-connectivity, background 0) + remove_small_objects (bincount < min_size removed) -> 0 / 255 uint8
    (background_removal.py:34-36)."""
    from scipy import ndimage

    labels, _ = ndimage.label(binary > 0, structure=np.ones((3, 3), dtype=int))
    sizes = np.bincount(labels.ravel())
    keep = sizes >= min_size
    keep[0] = False
    return keep[labels].astype(np.uint8) * 255


def refine_mask(mask: np.ndarray, min_size: int = 200) -> np.ndarray:
    """refine_mask (background_removal.py:20-38)."""
    _, binary = otsu_cv2(mask)
    return filter_components(binary, min_size)


def remove_background(sd: dict, image: np.ndarray, model_size: tuple, refine: bool = True, min_size: int = 200,
                      device="cpu") -> dict:
    """BackgroundRemover.forward (background_removal.py:84-112) -> dict(soft = sigmoid(d1), mask (uint8), rgba)."""
    with torch.no_grad():
        soft = rmbg_forward(sd, preprocess(image, model_size, device))
    mask = postprocess_mask(soft, image.shape[:2])
    alpha = refine_mask(mask, min_size) if refine else mask
    return dict(soft=soft[0, 0].cpu(), mask=mask, rgba=np.concatenate([image, alpha[:, :, None]], axis=2))


# ---- the kernels' operation order (numpy fp32) -----------------------------------------------------------------------------
def _taps(in_size: int, out_size: int):
    f = np.float32
    scale = f(in_size) / f(out_size)
    src = (scale * (np.arange(out_size, dtype=f) + f(0.5))).astype(f) - f(0.5)
    src = np.maximum(src.astype(f), f(0))
    i0 = src.astype(np.int64)
    i1 = i0 + (i0 < in_size - 1)
    l1 = (src - i0.astype(f)).astype(f)
    return i0, i1, (f(1) - l1).astype(f), l1


def bilinear_np(src: np.ndarray, out_h: int, out_w: int) -> np.ndarray:
    """(h, w, c) fp32 -> (out_h, out_w, c): h0 (w0 x00 + w1 x01) + h1 (w0 x10 + w1 x11), every operation rounded in fp32
    (csrc/rmbg.cu bilinear_tap / bilinear_mix)."""
    src = np.asarray(src, dtype=np.float32)
    y0, y1, hy0, hy1 = _taps(src.shape[0], out_h)
    x0, x1, wx0, wx1 = _taps(src.shape[1], out_w)
    wx0, wx1 = wx0[None, :, None], wx1[None, :, None]
    top = (wx0 * src[y0][:, x0]).astype(np.float32) + (wx1 * src[y0][:, x1]).astype(np.float32)
    bot = (wx0 * src[y1][:, x0]).astype(np.float32) + (wx1 * src[y1][:, x1]).astype(np.float32)
    return (hy0[:, None, None] * top).astype(np.float32) + (hy1[:, None, None] * bot).astype(np.float32)


def refine_rgba_restated(rgb: np.ndarray, mask: np.ndarray, refine: bool = True, min_size: int = 200) -> np.ndarray:
    """What amb_rmbg_refine_rgba writes, from the restated Otsu and the scipy component filter."""
    if refine:
        t = otsu_threshold(np.bincount(mask.ravel(), minlength=256))
        alpha = filter_components((mask > t).astype(np.uint8), min_size)
    else:
        alpha = mask
    return np.concatenate([rgb, alpha[:, :, None]], axis=2)


__all__ = ["make_state_dict", "rmbg_forward", "preprocess", "postprocess_mask", "refine_mask", "remove_background",
           "otsu_threshold", "otsu_cv2", "filter_components", "bilinear_np", "refine_rgba_restated", "synthetic_frame",
           "IGNORED_HEADS"]
