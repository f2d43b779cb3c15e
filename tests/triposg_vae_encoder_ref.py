"""Restatements used by the TripoSG VAE encoder tests (not collected by pytest).

  fps_numpy                 farthest-point sampling with the semantics of csrc/point_sampling.cu: fp32 distances
                            ((dx*dx) + (dy*dy)) + (dz*dz), each operation rounded on its own, running minimum from +inf,
                            argmax with ties to the lowest index.
  encode_fp32               fp32 restatement of TripoSGVAEModel._encode after the point sampling (autoencoder_kl_triposg.py:
                            26-87,439-457; DiTBlock of triposg_transformer.py; TripoSGAttnProcessor2_0's head-interleaved
                            splits), pinned against the reference module by tests/golden/triposg_vae_encoder_tiny.pt.
  make_encoder_state_dict   seeded, bf16-representable weights under TripoSGVAEModel's encoder-side keys.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

# LayerNorm rows of the CUDA path are >= 256 wide, hence width 256 (4 heads x 64) for the tiny encoder; the reference model
# of the golden also carries a decoder, 512 wide (4 heads x 128), 1 layer, unused here.
TINY = dict(width_encoder=256, num_attention_heads=4, num_layers_encoder=2, width_decoder=512, num_layers_decoder=1,
            latent_channels=64, embed_frequency=8)


def fps_numpy(xyz: np.ndarray, k: int, start: int) -> np.ndarray:
    """(N, 3) points -> (k,) int64 indices, the first `start`."""
    x = np.ascontiguousarray(xyz, dtype=np.float32)
    d = np.full(x.shape[0], np.inf, dtype=np.float32)
    out = np.empty(k, dtype=np.int64)
    sel = int(start)
    if k:
        out[0] = sel
    for r in range(1, k):
        diff = x - x[sel]
        e = (diff[:, 0] * diff[:, 0] + diff[:, 1] * diff[:, 1]) + diff[:, 2] * diff[:, 2]
        np.minimum(d, e, out=d)
        sel = int(np.argmax(d))
        out[r] = sel
    return out


def make_encoder_state_dict(width=512, heads=8, layers=8, latent_channels=64, embed_frequency=8, seed=0) -> dict:
    g = torch.Generator().manual_seed(seed)
    D, rs = width, 1.0 / math.sqrt(layers + 1)

    def lin(o, i, s=1.0):
        return ((torch.rand(o, i, generator=g) * 2 - 1) * s / math.sqrt(i)).to(torch.bfloat16).float()

    def vec(n, lo, hi):
        return (torch.rand(n, generator=g) * (hi - lo) + lo).to(torch.bfloat16).float()

    in_dim = 3 * (2 * embed_frequency + 1) + 3
    sd = {"encoder.proj_in.weight": lin(D, in_dim), "encoder.proj_in.bias": vec(D, -0.1, 0.1),
          "encoder.norm_out.weight": vec(D, 0.8, 1.2), "encoder.norm_out.bias": vec(D, -0.1, 0.1),
          "quant.weight": lin(2 * latent_channels, D), "quant.bias": vec(2 * latent_channels, -0.1, 0.1)}
    for i in range(layers + 1):
        p = f"encoder.blocks.{i}."
        a = "attn2" if i == 0 else "attn1"
        for n in ("norm2" if i == 0 else "norm1", "norm3"):
            sd[p + n + ".weight"], sd[p + n + ".bias"] = vec(D, 0.8, 1.2), vec(D, -0.1, 0.1)
        if i == 0:
            sd[p + "attn2.norm_cross.weight"], sd[p + "attn2.norm_cross.bias"] = vec(D, 0.8, 1.2), vec(D, -0.1, 0.1)
        for n in ("to_q", "to_k", "to_v"):
            sd[p + f"{a}.{n}.weight"] = lin(D, D)
        sd[p + f"{a}.to_out.0.weight"], sd[p + f"{a}.to_out.0.bias"] = lin(D, D, rs), vec(D, -0.02, 0.02)
        sd[p + "ff.net.0.proj.weight"], sd[p + "ff.net.0.proj.bias"] = lin(4 * D, D), vec(4 * D, -0.02, 0.02)
        sd[p + "ff.net.2.weight"], sd[p + "ff.net.2.bias"] = lin(D, 4 * D, rs), vec(D, -0.02, 0.02)
    return sd


def _ln(x, sd, name):
    return F.layer_norm(x, (x.shape[-1],), sd[name + ".weight"], sd[name + ".bias"], 1e-5)


def _embed(pts, embed_frequency):
    xyz = pts[..., :3]
    freqs = 2.0 ** torch.arange(embed_frequency, dtype=torch.float32, device=pts.device)
    emb = (xyz[..., None] * freqs).view(*xyz.shape[:-1], -1)
    return torch.cat([xyz, emb.sin(), emb.cos(), pts[..., 3:]], dim=-1)


def _ff(h, sd, p):
    hn = _ln(h, sd, p + "norm3")
    return h + (F.gelu(hn @ sd[p + "ff.net.0.proj.weight"].t() + sd[p + "ff.net.0.proj.bias"]) @ sd[p + "ff.net.2.weight"].t()
                + sd[p + "ff.net.2.bias"])


@torch.no_grad()
def encode_fp32(sd: dict, surface: torch.Tensor, sampled: torch.Tensor, heads: int, layers: int,
                embed_frequency: int = 8) -> torch.Tensor:
    """(B, N, 6) surface, (B, T, 6) sampled rows -> (B, T, 2C) `quant` output, fp32 on surface's device."""
    dev = surface.device
    sd = {k: v.to(device=dev, dtype=torch.float32) for k, v in sd.items() if k.startswith(("encoder.", "quant."))}
    B = surface.shape[0]
    x_kv = _embed(surface.float(), embed_frequency)
    x_q = _embed(sampled.to(dev, torch.float32), embed_frequency)
    h = x_q @ sd["encoder.proj_in.weight"].t() + sd["encoder.proj_in.bias"]
    ctx = x_kv @ sd["encoder.proj_in.weight"].t() + sd["encoder.proj_in.bias"]
    p = "encoder.blocks.0."
    q = _ln(h, sd, p + "norm2") @ sd[p + "attn2.to_q.weight"].t()
    c = _ln(ctx, sd, p + "attn2.norm_cross")
    kv = torch.cat([c @ sd[p + "attn2.to_k.weight"].t(), c @ sd[p + "attn2.to_v.weight"].t()], dim=-1)
    dh = kv.shape[-1] // heads // 2
    k, v = (t.transpose(1, 2) for t in kv.view(B, -1, heads, 2 * dh).split(dh, dim=-1))
    q = q.view(B, -1, heads, dh).transpose(1, 2)
    o = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B, -1, heads * dh)
    h = _ff(h + (o @ sd[p + "attn2.to_out.0.weight"].t() + sd[p + "attn2.to_out.0.bias"]), sd, p)
    for i in range(1, layers + 1):
        p = f"encoder.blocks.{i}."
        hn = _ln(h, sd, p + "norm1")
        qkv = torch.cat([hn @ sd[p + f"attn1.to_{n}.weight"].t() for n in "qkv"], dim=-1)
        dh = qkv.shape[-1] // heads // 3
        q, k, v = (t.transpose(1, 2) for t in qkv.view(B, -1, heads, 3 * dh).split(dh, dim=-1))
        o = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B, -1, heads * dh)
        h = _ff(h + (o @ sd[p + "attn1.to_out.0.weight"].t() + sd[p + "attn1.to_out.0.bias"]), sd, p)
    return _ln(h, sd, "encoder.norm_out") @ sd["quant.weight"].t() + sd["quant.bias"]


def posterior_sample(params: torch.Tensor, eps: torch.Tensor) -> torch.Tensor:
    """DiagonalGaussianDistribution(params, feature_dim=-1).sample() with the given eps (vae.py:8-36)."""
    mean, logvar = params.chunk(2, dim=-1)
    return mean + torch.exp(0.5 * logvar.clamp(-30.0, 20.0)) * eps


def sphere_surface(n: int, seed: int, radius: float = 0.8) -> torch.Tensor:
    """(1, n, 6) fp32 points on a sphere with their outward unit normals."""
    g = torch.Generator().manual_seed(seed)
    nrm = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1)
    return torch.cat([nrm * radius, nrm], dim=-1)[None]
