"""`B200BackgroundRemover`: the reference's `BackgroundRemover` (actionmesh/preprocessing/background_removal.py) on this
library's kernels, a drop-in for the pipeline's `background_removal=` argument.

BriaRMBG (third_party/TripoSG/scripts/briarmbg.py, RMBG-1.4) runs as a launch program: every 3x3 convolution is an im2col
into the split-bf16 operand (ops.rmbg_im2col_split) followed by one fp32-accumulating GEMM (ops.gemm) with BatchNorm folded
into the weights, ReLU (act 2) and the RSU residual in its epilogue; pooling, resampling, the side1 mask head and the
refinement (Otsu, 8-connected components, small-object removal) are kernels of csrc/rmbg.cu.  A frame is enqueued without a
host synchronisation; the only one is the final RGBA copy.  DESIGN.md §17 gives the precision argument and the semantics.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from . import ops
from ._lib import AmbError
from .module import B200Module, read_weights

BN_EPS = 1e-5
# (stage, RSU depth (0: RSU-4F), in, mid, out channels) in forward order (briarmbg.py:364-386)
ENCODER = (("stage1", 7, 64, 32, 64), ("stage2", 6, 64, 32, 128), ("stage3", 5, 128, 64, 256), ("stage4", 4, 256, 128, 512),
           ("stage5", 0, 512, 256, 512), ("stage6", 0, 512, 256, 512))
DECODER = (("stage5d", 0, 1024, 256, 512), ("stage4d", 4, 1024, 128, 256), ("stage3d", 5, 512, 64, 128),
           ("stage2d", 6, 256, 32, 64), ("stage1d", 7, 128, 16, 64))
IGNORED_HEADS = ("side2", "side3", "side4", "side5", "side6")  # never reach result[0][0] (background_removal.py:104-106)


def _pad64(n: int) -> int:
    return (n + 63) // 64 * 64


def rsu_convs(depth: int, cin: int, mid: int, cout: int) -> list[tuple[str, int, int, int]]:
    """(name, in channels, out channels, dilation) of every REBNCONV of an RSU-`depth` block (RSU-4F for depth 0), in
    forward order (briarmbg.py:37-328)."""
    convs = [("rebnconvin", cin, cout, 1)]
    if depth == 0:
        convs += [("rebnconv1", cout, mid, 1), ("rebnconv2", mid, mid, 2), ("rebnconv3", mid, mid, 4), ("rebnconv4", mid, mid, 8),
                  ("rebnconv3d", 2 * mid, mid, 4), ("rebnconv2d", 2 * mid, mid, 2), ("rebnconv1d", 2 * mid, cout, 1)]
        return convs
    convs.append(("rebnconv1", cout, mid, 1))
    convs += [(f"rebnconv{i}", mid, mid, 1) for i in range(2, depth)]
    convs.append((f"rebnconv{depth}", mid, mid, 2))
    convs += [(f"rebnconv{i}d", 2 * mid, mid, 1) for i in range(depth - 1, 1, -1)]
    convs.append(("rebnconv1d", 2 * mid, cout, 1))
    return convs


def conv_layers() -> list[tuple[str, int, int, int, bool]]:
    """(key prefix, in, out, dilation, has BatchNorm) of every convolution that runs on the GEMM, in forward order."""
    layers = [("conv_in", 3, 64, 1, False)]
    for stage, depth, cin, mid, cout in ENCODER + DECODER:
        layers += [(f"{stage}.{name}", i, o, d, True) for name, i, o, d in rsu_convs(depth, cin, mid, cout)]
    return layers


def fold_conv(sd: dict, prefix: str, bn: bool) -> tuple[torch.Tensor, torch.Tensor]:
    """(weight (O, I, 3, 3), bias (O,)) in fp64 with the eval-mode BatchNorm folded in: s = gamma / sqrt(var + eps),
    W' = s W, b' = s (b - mean) + beta (briarmbg.py:24)."""
    w, b = sd[f"{prefix}.weight"].double(), sd[f"{prefix}.bias"].double()
    if bn:
        bp = prefix.replace("conv_s1", "bn_s1")
        s = sd[f"{bp}.weight"].double() / torch.sqrt(sd[f"{bp}.running_var"].double() + BN_EPS)
        w = w * s[:, None, None, None]
        b = (b - sd[f"{bp}.running_mean"].double()) * s + sd[f"{bp}.bias"].double()
    return w, b


def pack_conv(w: torch.Tensor, b: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """fp64 (O, I, 3, 3) weight and (O,) bias -> (N_pad, 3 K_pad) bf16 in split3's weight layout [hi | hi | lo] of the fp32
    (O, ky, kx, I) rows zero-padded to N_pad = pad64(O), K_pad = pad64(9 I), and the (N_pad,) fp32 bias."""
    O, I = w.shape[:2]
    k = 9 * I
    wm = torch.zeros(_pad64(O), _pad64(k), dtype=torch.float32, device=w.device)
    wm[:O, :k] = w.permute(0, 2, 3, 1).reshape(O, k).float()
    hi = wm.to(torch.bfloat16)
    lo = (wm - hi.float()).to(torch.bfloat16)
    bias = torch.zeros(_pad64(O), dtype=torch.float32, device=w.device)
    bias[:O] = b.float()
    return torch.cat([hi, hi, lo], 1).contiguous(), bias


def expected_keys() -> set:
    keys = set()
    for prefix, _, _, _, bn in conv_layers():
        if bn:
            keys |= {f"{prefix}.conv_s1.weight", f"{prefix}.conv_s1.bias"}
            keys |= {f"{prefix}.bn_s1.{n}" for n in ("weight", "bias", "running_mean", "running_var")}
        else:
            keys |= {f"{prefix}.weight", f"{prefix}.bias"}
    return keys | {"side1.weight", "side1.bias"}


def _ignored(key: str) -> bool:
    return key.endswith(".num_batches_tracked") or key.split(".")[0] in IGNORED_HEADS


class _Workspace:
    """Every buffer of one model input size, allocated on first use and reused by later frames."""

    def __init__(self, device):
        self.device = device
        self.bufs: dict = {}
        self.frames: dict = {}  # frame size -> (mask-head tensors, refinement tensors)

    def get(self, name: str, shape: tuple, dtype=torch.float32) -> torch.Tensor:
        t = self.bufs.get(name)
        if t is None or tuple(t.shape) != tuple(shape):
            t = self.bufs[name] = torch.empty(shape, dtype=dtype, device=self.device)
        return t

    def col(self, rows: int, cols: int) -> torch.Tensor:
        """The shared im2col operand: grown to the largest convolution, viewed as (rows, cols)."""
        t = self.bufs.get("im2col")
        if t is None or t.numel() < rows * cols:
            self.bufs.pop("im2col", None)
            t = self.bufs["im2col"] = torch.empty(rows * cols, dtype=torch.bfloat16, device=self.device)
        return t[:rows * cols].view(rows, cols)


class B200BackgroundRemover(B200Module):
    """RMBG-1.4 background removal with the reference's surface: `forward(image)` on an (H, W, 3) uint8 array returns the
    (H, W, 4) RGBA array, `process_image(s)` on PIL images returns RGBA images (frames with a valid alpha mask are returned
    as they are, the same object)."""

    def __init__(self, rmbg_weights_dir: Optional[str] = None, model_input_size: tuple = (1024, 1024)):
        super().__init__()
        self.model_input_size = tuple(int(v) for v in model_input_size)
        if len(self.model_input_size) != 2 or min(self.model_input_size) < 1:
            raise AmbError(f"model_input_size must be two positive sizes, got {model_input_size}")
        self._ws: dict = {}
        if rmbg_weights_dir is not None:
            self.to("cuda")
            self.load_state_dict(read_weights(rmbg_weights_dir, self.weight_files))

    def _after_to(self, moved: bool) -> None:
        if moved:
            self._ws = {}

    def _pack_state_dict(self, sd: dict, device) -> dict:
        """BriaRMBG's state dict (its own key names) -> per convolution `<prefix>.w` (split weight) and `<prefix>.b`, plus
        `side1` (577,) = the (ky, kx, c) weights and the bias.  side2-side6 and num_batches_tracked are ignored; any other
        unknown or missing key raises."""
        want = expected_keys()
        unknown = sorted(k for k in sd if k not in want and not _ignored(k))
        missing = sorted(want - set(sd))
        if unknown or missing:
            raise AmbError(f"B200BackgroundRemover: unexpected keys {unknown[:5]}, missing keys {missing[:5]}")
        w = {}
        for prefix, cin, cout, _, bn in conv_layers():
            key = f"{prefix}.conv_s1" if bn else prefix
            wt = sd[f"{key}.weight"]
            if tuple(wt.shape) != (cout, cin, 3, 3):
                raise AmbError(f"{key}.weight: expected {(cout, cin, 3, 3)}, got {tuple(wt.shape)}")
            wp, bp = pack_conv(*fold_conv(sd, key, bn))
            w[f"{prefix}.w"], w[f"{prefix}.b"] = wp.to(device), bp.to(device)
        s1 = sd["side1.weight"]
        if tuple(s1.shape) != (1, 64, 3, 3):
            raise AmbError(f"side1.weight: expected (1, 64, 3, 3), got {tuple(s1.shape)}")
        w["side1"] = torch.cat([s1.float().permute(0, 2, 3, 1).reshape(-1), sd["side1.bias"].float().reshape(1)]).to(device)
        return w

    # ---- launch program ----------------------------------------------------------------------------------------------
    def _conv(self, ws: _Workspace, prefix: str, sources: list, h: int, w: int, *, dilation: int = 1, stride: int = 1,
              act: int = 2, residual: Optional[torch.Tensor] = None) -> torch.Tensor:
        wt, b = self._w[f"{prefix}.w"], self._w[f"{prefix}.b"]
        oh, ow = ops.conv3x3_out(h, stride, dilation, dilation), ops.conv3x3_out(w, stride, dilation, dilation)
        col = ws.col(oh * ow, wt.shape[1])
        ops.rmbg_im2col_split(sources, h, w, col, stride=stride, pad=dilation, dilation=dilation)
        out = ws.get(prefix, (oh * ow, wt.shape[0]))
        return ops.gemm(col, wt, out, bias=b, act=act, residual=residual, tag="rmbg_conv")

    @staticmethod
    def _pool(ws: _Workspace, name: str, x: torch.Tensor, h: int, w: int, c: int):
        oh, ow = (h + 1) // 2, (w + 1) // 2
        return ops.rmbg_maxpool2(x, h, w, c, ws.get(name, (oh * ow, c))), oh, ow

    @staticmethod
    def _upsample(ws: _Workspace, name: str, x: torch.Tensor, h: int, w: int, c: int, oh: int, ow: int) -> torch.Tensor:
        return ops.rmbg_upsample(x, h, w, c, ws.get(name, (oh * ow, c)), oh, ow)

    def _rsu(self, ws: _Workspace, stage: str, depth: int, mid: int, cout: int, sources: list, h: int, w: int) -> torch.Tensor:
        """RSU-`depth` (RSU-4F for 0) at (h, w): returns hx1d + hxin (briarmbg.py:74-116, 312-328)."""
        conv = lambda name, srcs, d=1, res=None: self._conv(ws, f"{stage}.{name}", srcs, h_, w_, dilation=d, residual=res)
        h_, w_ = h, w
        hxin = conv("rebnconvin", sources)
        if depth == 0:
            hx1 = conv("rebnconv1", [(hxin, cout)])
            hx2 = conv("rebnconv2", [(hx1, mid)], 2)
            hx3 = conv("rebnconv3", [(hx2, mid)], 4)
            hx4 = conv("rebnconv4", [(hx3, mid)], 8)
            d = conv("rebnconv3d", [(hx4, mid), (hx3, mid)], 4)
            d = conv("rebnconv2d", [(d, mid), (hx2, mid)], 2)
            return conv("rebnconv1d", [(d, mid), (hx1, mid)], 1, hxin)
        enc, sizes = [], []
        x, xc = hxin, cout
        for i in range(1, depth):
            hx = conv(f"rebnconv{i}", [(x, xc)])
            enc.append(hx)
            sizes.append((h_, w_))
            if i < depth - 1:
                x, h_, w_ = self._pool(ws, f"{stage}.pool{i}", hx, h_, w_, mid)
                xc = mid
        d = conv(f"rebnconv{depth}", [(enc[-1], mid)], 2)
        for i in range(depth - 1, 0, -1):
            h_, w_ = sizes[i - 1]
            d = conv(f"rebnconv{i}d", [(d, mid), (enc[i - 1], mid)], 1, hxin if i == 1 else None)
            if i > 1:
                d = self._upsample(ws, f"{stage}.up{i}", d, h_, w_, mid, *sizes[i - 2])
        return d

    def _network(self, ws: _Workspace, x: torch.Tensor, sh: int, sw: int) -> tuple[torch.Tensor, int, int]:
        """BriaRMBG.forward (briarmbg.py:397-441) on the (sh, sw, 3) preprocessed input -> (hx1d, its height, width)."""
        hc, wc = ops.conv3x3_out(sh, 2, 1, 1), ops.conv3x3_out(sw, 2, 1, 1)
        hxin = self._conv(ws, "conv_in", [(x.view(sh * sw, 3), 3)], sh, sw, stride=2, act=0)
        feats, sizes = [], []
        h, w, src = hc, wc, [(hxin, 64)]
        for i, (stage, depth, cin, mid, cout) in enumerate(ENCODER):
            hx = self._rsu(ws, stage, depth, mid, cout, src, h, w)
            feats.append((hx, cout))
            sizes.append((h, w))
            if i < len(ENCODER) - 1:
                p, h, w = self._pool(ws, f"pool{i + 1}{i + 2}", hx, h, w, cout)
                src = [(p, cout)]
        d, dc = feats[-1]
        for j, (stage, depth, cin, mid, cout) in enumerate(DECODER):
            skip, sc = feats[-2 - j]
            th, tw = sizes[-2 - j]
            up = self._upsample(ws, f"{stage}.in", d, h, w, dc, th, tw)
            h, w = th, tw
            d, dc = self._rsu(ws, stage, depth, mid, cout, [(up, dc), (skip, sc)], h, w), cout
        return d, h, w

    def _run(self, rgb: torch.Tensor, refine: bool = True, min_size: int = 200) -> tuple[torch.Tensor, dict]:
        """(H, W, 3) uint8 CUDA frame -> ((H, W, 4) uint8 RGBA on the device, the mask head's tensors: logits, soft =
        sigmoid(d1), resized, mask).  Everything is enqueued on the current stream; nothing is read back."""
        self._check_loaded()
        sh, sw = self.model_input_size
        ws = self._ws.get((sh, sw))
        if ws is None:
            ws = self._ws[(sh, sw)] = _Workspace(self._device)
        x = ops.rmbg_resize_input(rgb, ws.get("input", (sh, sw, 3)))
        hx1d, h, w = self._network(ws, x, sh, sw)
        H, W = rgb.shape[0], rgb.shape[1]
        head_work, refine_work = ws.frames.setdefault((H, W), ({}, {}))
        head = ops.rmbg_mask_head(hx1d, h, w, self._w["side1"], (sh, sw), (H, W), head_work)
        rgba = ops.rmbg_refine_rgba(rgb, head["mask"], refine, min_size, work=refine_work)
        return rgba, head

    # ---- the reference's surface -------------------------------------------------------------------------------------
    @ops.on_device
    @torch.no_grad()
    def forward(self, image: np.ndarray, refine: bool = True, min_size: int = 200) -> np.ndarray:
        """(H, W, 3) uint8 RGB array -> (H, W, 4) uint8 RGBA array whose alpha is the (refined) foreground mask
        (background_removal.py:84-112)."""
        image = np.asarray(image)
        if image.dtype != np.uint8 or image.ndim != 3 or image.shape[2] != 3 or min(image.shape[:2]) < 1:
            raise AmbError(f"B200BackgroundRemover: expected an (H, W, 3) uint8 image, got {image.shape} {image.dtype}")
        rgb = torch.from_numpy(np.ascontiguousarray(image)).to(self._device)
        rgba, _ = self._run(rgb, refine, min_size)
        return rgba.cpu().numpy()

    __call__ = forward

    @staticmethod
    def _has_a_valid_alpha_mask(image, threshold: int = 127) -> bool:
        """RGBA with at least 1 % of the pixels on each side of alpha > threshold (background_removal.py:114-128,
        image_processor.py:15-23); a host-side count, so a valid frame launches nothing."""
        if image.mode != "RGBA":
            return False
        alpha = np.asarray(image.getchannel("A"))
        min_count = int(alpha.size * 0.01)
        fg = int(np.count_nonzero(alpha > threshold))
        return alpha.size - fg >= min_count and fg >= min_count

    def process_image(self, image):
        """PIL image -> the same image when it already has a valid alpha mask, else the RGBA image with the background
        removed (background_removal.py:130-145)."""
        from PIL import Image

        if self._has_a_valid_alpha_mask(image):
            return image
        return Image.fromarray(self.forward(np.array(image.convert("RGB"))), "RGBA")

    def process_images(self, images: list) -> list:
        return [self.process_image(image) for image in images]
