"""B200ImageEncoder — DinoV2-L/14 frame encoder behind the reference's ImageEncoder surface.

Mirrors actionmesh/model/image_encoder.py:16-55: constructor kwargs `pretrained_dino_feature_extractor`,
`pretrained_dino_model`; `.encode_images(list[PIL]) -> (T, 257, 1024) fp32`; `.device`, `.eval()`, `.to()`.
The transformer (HF `Dinov2Model`, transformers/models/dinov2/modeling_dinov2.py: patch-embed conv, CLS + interpolated
position embeddings, 24 x [LN, MHA(16 heads, d_h 64), LayerScale, LN, MLP GELU, LayerScale], final LN) runs on the sm_90a
kernels: patchify (im2col) -> wgmma GEMM, LayerNorm, fused-QKV wgmma GEMM, wgmma flash attention (head_dim 64),
GEMM epilogues with bias / GELU / LayerScale / fp32 residual.

Precision.  The reference runs DinoV2 in fp32, outside autocast (pipeline.py:664-667), so the default here is fp32-grade
(`precision="fp32"`): every linear runs on the tensor cores with three-way split bf16 operands (x = hi + lo; activations
[hi|lo|hi], weights [hi|hi|lo] along K, fp32 accumulation: all products but lo·lo, relative error ~2^-16 — the machinery of
the Stage-II query path), activations and the residual stream stay fp32 between kernels, and the 257-token attention runs in
fp32 on the CUDA cores (csrc/attention_small.cu).  The encoder is 2.5 TFLOP per clip against 16 400 for the denoise, so
3x its GEMM work is invisible.  `precision="bf16"` keeps the round-1 path (bf16 operands, wgmma flash attention at
head_dim 64; last_hidden_state within 1e-2 of fp32).

Image preprocessing (HF BitImageProcessor in the reference: bicubic resize to 256, centre crop 224, 1/255 rescale, ImageNet
mean/std) runs on the GPU with the semantics of the reference's pinned transformers<5 / Pillow path, bit-exact on the uint8
image (actionmesh_b200/preprocess.py); `image_preprocess_dino` keeps the HF object as the source of the configuration.
"""
from __future__ import annotations

import json
import math
import os
from typing import List, Optional

import torch

from . import blocks, ops
from ._lib import AmbError
from .module import B200Module, read_weights

IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)


def default_preprocessor():
    """facebook/dinov2-large preprocessor_config (hub file, not available offline): shortest_edge 256 bicubic, centre
    crop 224, rescale 1/255, ImageNet normalisation."""
    from transformers import BitImageProcessor

    return BitImageProcessor(do_resize=True, size={"shortest_edge": 256}, resample=3, do_center_crop=True,
                             crop_size={"height": 224, "width": 224}, do_rescale=True, rescale_factor=1 / 255.0,
                             do_normalize=True, image_mean=list(IMAGENET_MEAN), image_std=list(IMAGENET_STD),
                             do_convert_rgb=True)


def hf_dinov2_arguments(model_dir: str, feature_extractor_dir: str) -> dict:
    """B200ImageEncoder's shape arguments for an HF `Dinov2Model` directory and its `BitImageProcessor` directory.

    `Dinov2Config` does not name things the way the constructor does, so `B200Module.from_pretrained`'s match by name would
    go wrong: `num_hidden_layers` / `num_attention_heads` are `num_layers` / `num_heads`, and its `image_size` is the grid
    the position embeddings were trained at (518 for dinov2-large), not the input size.  The input size is the feature
    extractor's crop, the size `B200ImagePreprocessor.from_hf` produces; it must be square and a multiple of the patch."""
    from transformers import BitImageProcessor

    from .preprocess import B200ImagePreprocessor

    for d, name in ((model_dir, "config.json"), (feature_extractor_dir, "preprocessor_config.json")):
        if not os.path.isfile(os.path.join(d, name)):
            raise AmbError(f"B200ImageEncoder: {os.path.join(d, name)} not found")
    with open(os.path.join(model_dir, "config.json")) as f:
        cfg = json.load(f)
    if cfg.get("use_swiglu_ffn", False) or cfg.get("hidden_act", "gelu") != "gelu":
        raise AmbError("B200ImageEncoder: only DinoV2's GELU MLP is supported")
    patch = int(cfg.get("patch_size", 14))
    ch, cw = B200ImagePreprocessor.from_hf(BitImageProcessor.from_pretrained(feature_extractor_dir)).crop_size
    if ch != cw or ch % patch:
        raise AmbError(f"B200ImageEncoder: the crop {ch}x{cw} of {feature_extractor_dir} must be square and a multiple of "
                       f"patch_size {patch}")
    return dict(hidden_size=int(cfg.get("hidden_size", 1024)), num_layers=int(cfg["num_hidden_layers"]),
                num_heads=int(cfg["num_attention_heads"]), patch_size=patch, image_size=ch,
                mlp_ratio=int(cfg.get("mlp_ratio", 4)), layer_norm_eps=float(cfg.get("layer_norm_eps", 1e-6)))


class B200ImageEncoder(B200Module):
    def __init__(self, pretrained_dino_feature_extractor: Optional[str] = None,
                 pretrained_dino_model: Optional[str] = None, *, hidden_size: int = 1024, num_layers: int = 24,
                 num_heads: int = 16, patch_size: int = 14, image_size: int = 224, mlp_ratio: int = 4,
                 layer_norm_eps: float = 1e-6, precision: str = "fp32"):
        self.hidden_size, self.num_layers, self.num_heads = hidden_size, num_layers, num_heads
        self.patch_size, self.image_size, self.mlp_ratio, self.eps = patch_size, image_size, mlp_ratio, layer_norm_eps
        if hidden_size // num_heads != 64 or hidden_size % 256:
            raise AmbError("B200ImageEncoder: head_dim must be 64 and hidden_size a multiple of 256")
        if precision not in ("fp32", "bf16"):
            raise AmbError("B200ImageEncoder: precision must be 'fp32' (reference-grade, default) or 'bf16'")
        self.precision = precision
        super().__init__()
        self._pending_sd = None
        self.image_preprocess_dino = None
        self._gpu_preprocess = None
        # A given path must be a local checkpoint directory (the reference downloads 'facebook/dinov2-large' into
        # pretrained_weights/dinov2 first, pipeline.py:75-78; there is no network here): a hub id or a missing directory is an
        # error NOW, not a silent fall-back to default preprocessing and unloaded weights.
        for what, path in (("pretrained_dino_feature_extractor", pretrained_dino_feature_extractor),
                           ("pretrained_dino_model", pretrained_dino_model)):
            if path is not None and not os.path.isdir(path):
                raise AmbError(f"B200ImageEncoder: {what}={path!r} is not a local directory (download the checkpoint "
                               "first, or pass None and call load_state_dict / init_random_)")
        if pretrained_dino_feature_extractor is not None:
            from transformers import BitImageProcessor
            self.image_preprocess_dino = BitImageProcessor.from_pretrained(pretrained_dino_feature_extractor)
        if self.image_preprocess_dino is None:
            self.image_preprocess_dino = default_preprocessor()
        if pretrained_dino_model is not None:
            self._pending_sd = read_weights(pretrained_dino_model, self.weight_files)

    @classmethod
    def from_hf_dirs(cls, model_dir: str, feature_extractor_dir: str, precision: str = "fp32", device="cuda"):
        """An HF `Dinov2Model` directory (config.json + weights) and its `BitImageProcessor` directory
        (preprocessor_config.json), loaded onto `device`; the constructor arguments are `hf_dinov2_arguments`'."""
        return cls(feature_extractor_dir, model_dir, precision=precision,
                   **hf_dinov2_arguments(model_dir, feature_extractor_dir)).to(device)

    def _after_to(self, moved: bool) -> None:
        """The weights of `pretrained_dino_model` are packed on the first `to()`."""
        if self._pending_sd is not None:
            self.load_state_dict(self._pending_sd)
            self._pending_sd = None

    # ---- weights (HF Dinov2Model state-dict keys)
    def _pack_state_dict(self, sd: dict, dev: torch.device) -> dict:
        sd = {k[len("dinov2."):] if k.startswith("dinov2.") else k: v for k, v in sd.items()}
        D, P = self.hidden_size, self.patch_size
        f32 = lambda k: sd[k].detach().to(device=dev, dtype=torch.float32)
        V = lambda k: blocks.V(sd[k], dev)
        if self.precision == "fp32":   # split operand [hi | hi | lo] along K (ops.split3, weight layout)
            W = lambda t: ops.split3(t.contiguous(), torch.empty(t.shape[0], 3 * t.shape[1], dtype=torch.bfloat16, device=dev),
                                     weight=True)
        else:
            W = lambda t: t.to(torch.bfloat16).contiguous()
        w = {}
        kreal = 3 * P * P
        self.kpad = (kreal + 63) // 64 * 64
        pw = torch.zeros(D, self.kpad, device=dev)
        pw[:, :kreal] = f32("embeddings.patch_embeddings.projection.weight").reshape(D, kreal)
        w["patch.w"], w["patch.b"] = W(pw), f32("embeddings.patch_embeddings.projection.bias").contiguous()
        # position embeddings interpolated once for the fixed 224x224 grid (modeling_dinov2 interpolate_pos_encoding:
        # bicubic, align_corners=False, fp32), CLS position kept; + cls token folded into row 0.
        pos = f32("embeddings.position_embeddings")[0]
        n_side_src = int(math.isqrt(pos.shape[0] - 1))
        g = self.image_size // P
        grid = pos[1:].reshape(1, n_side_src, n_side_src, D).permute(0, 3, 1, 2)
        if n_side_src != g:
            grid = torch.nn.functional.interpolate(grid, size=(g, g), mode="bicubic", align_corners=False)
        grid = grid.permute(0, 2, 3, 1).reshape(g * g, D)
        base = torch.cat([(f32("embeddings.cls_token")[0, 0] + pos[0])[None], grid], dim=0)  # (1+g*g, D)
        w["base"] = base.contiguous()
        for i in range(self.num_layers):
            p = f"encoder.layer.{i}."
            a = p + "attention.attention."
            w[p + "norm_s_attn.g"], w[p + "norm_s_attn.b"] = V(p + "norm1.weight"), V(p + "norm1.bias")
            w[p + "s.qkv"] = W(torch.cat([f32(a + "query.weight"), f32(a + "key.weight"), f32(a + "value.weight")], 0))
            w[p + "s.qkv.b"] = torch.cat([f32(a + "query.bias"), f32(a + "key.bias"), f32(a + "value.bias")], 0).contiguous()
            w[p + "s.o.w"], w[p + "s.o.b"] = W(f32(p + "attention.output.dense.weight")), V(p + "attention.output.dense.bias")
            w[p + "ls1"] = V(p + "layer_scale1.lambda1")
            w[p + "norm_ff.g"], w[p + "norm_ff.b"] = V(p + "norm2.weight"), V(p + "norm2.bias")
            w[p + "ff1.w"], w[p + "ff1.b"] = W(f32(p + "mlp.fc1.weight")), V(p + "mlp.fc1.bias")
            w[p + "ff2.w"], w[p + "ff2.b"] = W(f32(p + "mlp.fc2.weight")), V(p + "mlp.fc2.bias")
            w[p + "ls2"] = V(p + "layer_scale2.lambda1")
        w["ln.g"], w["ln.b"] = V("layernorm.weight"), V("layernorm.bias")
        return w

    @ops.on_device
    def init_random_(self, seed: int = 1235) -> None:
        """Synthetic DinoV2 weights with the HF key names (benchmarks only; no checkpoints offline)."""
        dev = self._device
        g = torch.Generator(device=dev).manual_seed(seed)
        D, P, F_ = self.hidden_size, self.patch_size, self.hidden_size * self.mlp_ratio

        def rnd(*shape, scale=0.02):
            return torch.randn(*shape, generator=g, device=dev) * scale

        sd = {"embeddings.cls_token": rnd(1, 1, D, scale=0.2),
              "embeddings.position_embeddings": rnd(1, 1 + 37 * 37, D, scale=0.2),
              "embeddings.patch_embeddings.projection.weight": rnd(D, 3, P, P),
              "embeddings.patch_embeddings.projection.bias": rnd(D),
              "layernorm.weight": torch.ones(D, device=dev), "layernorm.bias": torch.zeros(D, device=dev)}
        for i in range(self.num_layers):
            p_ = f"encoder.layer.{i}."
            for n in ("norm1", "norm2"):
                sd[p_ + n + ".weight"], sd[p_ + n + ".bias"] = torch.ones(D, device=dev), torch.zeros(D, device=dev)
            for n in ("query", "key", "value"):
                sd[p_ + f"attention.attention.{n}.weight"], sd[p_ + f"attention.attention.{n}.bias"] = rnd(D, D), rnd(D)
            sd[p_ + "attention.output.dense.weight"], sd[p_ + "attention.output.dense.bias"] = rnd(D, D), rnd(D)
            sd[p_ + "layer_scale1.lambda1"] = torch.full((D,), 0.5, device=dev)
            sd[p_ + "layer_scale2.lambda1"] = torch.full((D,), 0.5, device=dev)
            sd[p_ + "mlp.fc1.weight"], sd[p_ + "mlp.fc1.bias"] = rnd(F_, D), rnd(F_)
            sd[p_ + "mlp.fc2.weight"], sd[p_ + "mlp.fc2.bias"] = rnd(D, F_), rnd(D)
        self.load_state_dict(sd)

    # ---- encode
    @ops.on_device
    @torch.no_grad()
    def encode_images(self, images: List) -> torch.Tensor:
        """images: list of T PIL images -> context (T, 257, 1024) fp32 (image_encoder.py:38-55)."""
        if self._gpu_preprocess is None:
            from .preprocess import B200ImagePreprocessor

            self._gpu_preprocess = B200ImagePreprocessor.from_hf(self.image_preprocess_dino)
        return self.encode_pixel_values(self._gpu_preprocess.preprocess(images, self._device))

    @ops.on_device
    @torch.no_grad()
    def encode_pixel_values(self, pixel_values: torch.Tensor) -> torch.Tensor:
        """pixel_values (T,3,224,224) fp32 (host or device) -> last_hidden_state (T, 1+g*g, D) fp32."""
        self._check_loaded()
        w = self._w
        dev = self._device
        px = pixel_values.to(device=dev, dtype=torch.float32).contiguous()
        T = px.shape[0]
        D, H, P = self.hidden_size, self.num_heads, self.patch_size
        g = self.image_size // P
        L = 1 + g * g
        M = T * L
        F_ = D * self.mlp_ratio
        bf = torch.bfloat16
        x = w["base"].repeat(T, 1)                      # (M, D) fp32 residual stream: cls+pos rows (device copy)
        if self.precision == "fp32":
            return self._encode_fp32(px, x, T, L, M, F_)
        patches = ops.patchify(px, P, self.kpad)
        ops.gemm(patches, w["patch.w"], x, bias=w["patch.b"], residual=x, row_map=(g * g, L, 1))
        xn = torch.empty(M, D, dtype=bf, device=dev)
        qkv = torch.empty(M, 3 * D, dtype=bf, device=dev)
        att = torch.empty(M, D, dtype=bf, device=dev)
        hid = torch.empty(M, F_, dtype=bf, device=dev)
        for i in range(self.num_layers):
            p = f"encoder.layer.{i}."
            blocks.attention_half(w, p, x, xn, qkv, att, (T, L), H, eps=self.eps, bias=w[p + "s.qkv.b"], tag="gemm",
                                  attn_tag="attn_dino")
            blocks.output_half(w, p, "s", x, att, xn, hid, eps=self.eps, layer_scale=(w[p + "ls1"], w[p + "ls2"]), tag="gemm")
        out = torch.empty(M, D, dtype=torch.float32, device=dev)
        ops.layernorm(x, w["ln.g"], w["ln.b"], self.eps, out=out)
        return out.view(T, L, D)

    def _encode_fp32(self, px: torch.Tensor, x: torch.Tensor, T: int, L: int, M: int, F_: int) -> torch.Tensor:
        """The fp32-grade path: split-bf16 tensor-core GEMMs, fp32 activations, fp32 CUDA-core attention."""
        w, dev = self._w, self._device
        D, H, P = self.hidden_size, self.num_heads, self.patch_size
        g = self.image_size // P
        bf, f32 = torch.bfloat16, torch.float32
        # im2col of the stride-P patch convolution: a pure re-indexing of the fp32 pixels (columns ordered (c, py, px) like the
        # conv weight), zero-padded to the GEMM's K granularity
        cols = torch.zeros(T * g * g, self.kpad, dtype=f32, device=dev)
        cols[:, :3 * P * P] = px.reshape(T, 3, g, P, g, P).permute(0, 2, 4, 1, 3, 5).reshape(T * g * g, 3 * P * P)
        p3 = ops.split3(cols, torch.empty(T * g * g, 3 * self.kpad, dtype=bf, device=dev))
        ops.gemm(p3, w["patch.w"], x, bias=w["patch.b"], residual=x, row_map=(g * g, L, 1))
        t32 = torch.empty(M, D, dtype=f32, device=dev)
        a3 = torch.empty(M, 3 * D, dtype=bf, device=dev)
        qkv = torch.empty(M, 3 * D, dtype=f32, device=dev)
        att = torch.empty(M, D, dtype=f32, device=dev)
        hid = torch.empty(M, F_, dtype=f32, device=dev)
        h3 = torch.empty(M, 3 * F_, dtype=bf, device=dev)
        scale = 1.0 / math.sqrt(D // H)
        for i in range(self.num_layers):
            p = f"encoder.layer.{i}."
            ops.layernorm(x, w[p + "norm_s_attn.g"], w[p + "norm_s_attn.b"], self.eps, out=t32)
            ops.split3(t32, a3)
            ops.gemm(a3, w[p + "s.qkv"], qkv, bias=w[p + "s.qkv.b"])
            ops.attn_small_f32(qkv, T, L, H, scale, att, tag="attn_dino")
            ops.split3(att, a3)
            ops.gemm(a3, w[p + "s.o.w"], x, bias=w[p + "s.o.b"], col_scale=w[p + "ls1"], residual=x)
            ops.layernorm(x, w[p + "norm_ff.g"], w[p + "norm_ff.b"], self.eps, out=t32)
            ops.split3(t32, a3)
            ops.gemm(a3, w[p + "ff1.w"], hid, bias=w[p + "ff1.b"], act=1)
            ops.split3(hid, h3)
            ops.gemm(h3, w[p + "ff2.w"], x, bias=w[p + "ff2.b"], col_scale=w[p + "ls2"], residual=x)
        out = torch.empty(M, D, dtype=f32, device=dev)
        ops.layernorm(x, w["ln.g"], w["ln.b"], self.eps, out=out)
        return out.view(T, L, D)
