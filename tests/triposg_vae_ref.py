"""Restatements used by the TripoSG VAE / mesh-extraction tests (not collected by pytest).

  decode_fp32      fp32 restatement of TripoSGVAEModel.decode (autoencoder_kl_triposg.py:193-216,481-509, DiTBlock of
                   triposg_transformer.py:288-362, TripoSGAttnProcessor2_0's head-interleaved splits), pinned against the
                   reference module by tests/golden/triposg_vae_tiny.pt.
  make_state_dict  seeded, bf16-representable weights under TripoSGVAEModel's decoder-side keys.
  sphere / torus   analytic logit fields (positive inside) built from mul / add / sub only, each rounded on its own, so a
                   CPU and a GPU evaluation agree bit for bit.
  dmc_numpy        numpy restatement of the dual marching cubes of csrc/geometry.cu (vertex placement, patch table, quad
                   rules, winding, output order).  Project-authored and unpinned: the reference's DiffDMC (diso) is not
                   available to compare against.
"""
from __future__ import annotations

import math
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from gen_dmc_table import dmc_tables  # noqa: E402

TINY = dict(width_decoder=256, num_attention_heads=2, num_layers_decoder=2, latent_channels=64, embed_frequency=8)
BOUNDS = (-1.005, -1.005, -1.005, 1.005, 1.005, 1.005)


def make_state_dict(width=1024, heads=8, layers=16, latent_channels=64, embed_frequency=8, seed=0) -> dict:
    g = torch.Generator().manual_seed(seed)
    D, rs = width, 1.0 / math.sqrt(layers + 1)

    def lin(o, i, s=1.0):
        return ((torch.rand(o, i, generator=g) * 2 - 1) * s / math.sqrt(i)).to(torch.bfloat16).float()

    def vec(n, lo, hi):
        return (torch.rand(n, generator=g) * (hi - lo) + lo).to(torch.bfloat16).float()

    qdim = 3 * (2 * embed_frequency + 1)
    sd = {"post_quant.weight": lin(D, latent_channels), "post_quant.bias": vec(D, -0.1, 0.1),
          "decoder.proj_query.weight": lin(D, qdim), "decoder.proj_query.bias": vec(D, -0.1, 0.1),
          "decoder.norm_out.weight": vec(D, 0.8, 1.2), "decoder.norm_out.bias": vec(D, -0.1, 0.1),
          "decoder.proj_out.weight": lin(1, D), "decoder.proj_out.bias": vec(1, -0.1, 0.1)}
    for i in range(layers + 1):
        p = f"decoder.blocks.{i}."
        a = "attn2" if i == layers else "attn1"
        for n in ("norm2" if i == layers else "norm1", "norm3"):
            sd[p + n + ".weight"], sd[p + n + ".bias"] = vec(D, 0.8, 1.2), vec(D, -0.1, 0.1)
        if i == layers:
            sd[p + "attn2.norm_cross.weight"], sd[p + "attn2.norm_cross.bias"] = vec(D, 0.8, 1.2), vec(D, -0.1, 0.1)
        for n in ("to_q", "to_k", "to_v"):
            sd[p + f"{a}.{n}.weight"] = lin(D, D)
        sd[p + f"{a}.to_out.0.weight"], sd[p + f"{a}.to_out.0.bias"] = lin(D, D, rs), vec(D, -0.02, 0.02)
        sd[p + "ff.net.0.proj.weight"], sd[p + "ff.net.0.proj.bias"] = lin(4 * D, D), vec(4 * D, -0.02, 0.02)
        sd[p + "ff.net.2.weight"], sd[p + "ff.net.2.bias"] = lin(D, 4 * D, rs), vec(D, -0.02, 0.02)
    return sd


def _ln(x, sd, name):
    return F.layer_norm(x, (x.shape[-1],), sd[name + ".weight"], sd[name + ".bias"], 1e-5)


@torch.no_grad()
def decode_fp32(sd: dict, z: torch.Tensor, points: torch.Tensor, heads: int, layers: int, embed_frequency: int = 8,
                kv_cache: torch.Tensor = None, return_kv: bool = False):
    """(B, N, C) latents, (B, P, 3) points -> (B, P, 1) logits in fp32 on z's device (kv_cache: the trunk output)."""
    sd = {k: v.to(device=z.device, dtype=torch.float32) for k, v in sd.items()}
    if kv_cache is None:
        h = z.float() @ sd["post_quant.weight"].t() + sd["post_quant.bias"]
        B = h.shape[0]
        for i in range(layers):
            p = f"decoder.blocks.{i}."
            hn = _ln(h, sd, p + "norm1")
            qkv = torch.cat([hn @ sd[p + f"attn1.to_{n}.weight"].t() for n in "qkv"], dim=-1)
            dh = qkv.shape[-1] // heads // 3
            q, k, v = (t.transpose(1, 2) for t in qkv.view(B, -1, heads, 3 * dh).split(dh, dim=-1))
            o = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B, -1, heads * dh)
            h = h + (o @ sd[p + "attn1.to_out.0.weight"].t() + sd[p + "attn1.to_out.0.bias"])
            hn = _ln(h, sd, p + "norm3")
            h = h + (F.gelu(hn @ sd[p + "ff.net.0.proj.weight"].t() + sd[p + "ff.net.0.proj.bias"]) @ sd[p + "ff.net.2.weight"].t()
                     + sd[p + "ff.net.2.bias"])
        kv_cache = h
    B = points.shape[0]
    x = points.to(z.device, torch.float32)
    freqs = 2.0 ** torch.arange(embed_frequency, dtype=torch.float32, device=z.device)
    emb = (x[..., None] * freqs).view(*x.shape[:-1], -1)
    x = torch.cat([x, emb.sin(), emb.cos()], dim=-1) @ sd["decoder.proj_query.weight"].t() + sd["decoder.proj_query.bias"]
    p = f"decoder.blocks.{layers}."
    q = _ln(x, sd, p + "norm2") @ sd[p + "attn2.to_q.weight"].t()
    ctx = _ln(kv_cache, sd, p + "attn2.norm_cross")
    kv = torch.cat([ctx @ sd[p + "attn2.to_k.weight"].t(), ctx @ sd[p + "attn2.to_v.weight"].t()], dim=-1)
    dh = kv.shape[-1] // heads // 2
    k, v = (t.transpose(1, 2) for t in kv.view(B, -1, heads, 2 * dh).split(dh, dim=-1))
    q = q.view(B, -1, heads, dh).transpose(1, 2)
    o = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B, -1, heads * dh)
    x = x + (o @ sd[p + "attn2.to_out.0.weight"].t() + sd[p + "attn2.to_out.0.bias"])
    hn = _ln(x, sd, p + "norm3")
    x = x + (F.gelu(hn @ sd[p + "ff.net.0.proj.weight"].t() + sd[p + "ff.net.0.proj.bias"]) @ sd[p + "ff.net.2.weight"].t()
             + sd[p + "ff.net.2.bias"])
    out = -(_ln(x, sd, "decoder.norm_out") @ sd["decoder.proj_out.weight"].t() + sd["decoder.proj_out.bias"])
    return (out, kv_cache) if return_kv else out


# ---- analytic fields: xyz (P, 3) fp32 -> (P, 1) fp32 logits, positive inside ----------------------------------------------
SPHERE_R = 0.625
TORUS_R, TORUS_r = 0.5, 0.25


def sphere(xyz):
    """64 (R^2 - |x|^2); the factor keeps the |logit| < 0.95 band about a voxel wide at depth 8."""
    x, y, z = xyz[:, 0:1], xyz[:, 1:2], xyz[:, 2:3]
    return (SPHERE_R * SPHERE_R - (x * x + y * y + z * z)) * 64.0


def torus(xyz):
    """128 (4 R^2 (x^2 + y^2) - (|x|^2 + R^2 - r^2)^2): the implicit quartic of a torus around z."""
    x, y, z = xyz[:, 0:1], xyz[:, 1:2], xyz[:, 2:3]
    rho2 = x * x + y * y
    s = rho2 + z * z + (TORUS_R * TORUS_R - TORUS_r * TORUS_r)
    return (rho2 * (4.0 * TORUS_R * TORUS_R) - s * s) * 128.0


def sphere_distance(v):
    return np.abs(np.linalg.norm(v, axis=-1) - SPHERE_R)


def torus_distance(v):
    rho = np.linalg.norm(v[:, :2], axis=-1)
    return np.abs(np.sqrt((rho - TORUS_R) ** 2 + v[:, 2] ** 2) - TORUS_r)


def dense_grid(field, n: int, lo: float = -1.0, hi: float = 1.0) -> np.ndarray:
    """(n, n, n) fp32 grid of `field` at linspace(lo, hi, n) along each axis (x slowest)."""
    a = np.linspace(lo, hi, n, dtype=np.float32)
    xyz = np.stack(np.meshgrid(a, a, a, indexing="ij"), axis=-1).reshape(-1, 3)
    return field(torch.from_numpy(xyz)).numpy().reshape(n, n, n)


# ---- dual marching cubes --------------------------------------------------------------------------------------------------
_PATCH, _NPATCH = (np.array(t) for t in dmc_tables())


def _edge_corners(e):
    axis, u, v = e >> 2, e & 1, (e >> 1) & 1
    o0, o1 = (1, 2) if axis == 0 else ((0, 2) if axis == 1 else (0, 1))
    off = [0, 0, 0]
    off[o0], off[o1] = u, v
    c0 = off[0] | (off[1] << 1) | (off[2] << 2)
    return axis, o0, o1, u, v, c0, c0 | (1 << axis)


def dmc_numpy(grid: np.ndarray):
    """Same output as ops.dual_marching_cubes: vertices (V, 3) fp32 in grid-index units, faces (F, 3) int64."""
    g = np.ascontiguousarray(grid, dtype=np.float32)
    n = g.shape[0]
    m = n - 1
    corners = [g[(k & 1):(k & 1) + m, ((k >> 1) & 1):((k >> 1) & 1) + m, ((k >> 2) & 1):((k >> 2) & 1) + m] for k in range(8)]
    ok = np.ones((m, m, m), dtype=bool)
    case = np.zeros((m, m, m), dtype=np.int64)
    for k, c in enumerate(corners):
        ok &= np.isfinite(c)
        case |= (c > 0).astype(np.int64) << k
    case[~ok] = 0
    npatch = _NPATCH[case]
    voff = (np.cumsum(npatch.ravel()) - npatch.ravel()).reshape(m, m, m)
    nv = int(npatch.sum())
    s = np.zeros((nv, 3), dtype=np.float32)
    cnt = np.zeros(nv, dtype=np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        for e in range(12):
            axis, o0, o1, u, v, c0, c1 = _edge_corners(e)
            p = _PATCH[case, e]
            sel = p >= 0
            vid = (voff + p)[sel]
            a, b = corners[c0][sel], corners[c1][sel]
            t = (a / (a - b)).astype(np.float32)
            s[vid, axis] = s[vid, axis] + t
            s[vid, o0] = s[vid, o0] + np.float32(u)
            s[vid, o1] = s[vid, o1] + np.float32(v)
            cnt[vid] += 1
    cell_of_vertex = np.repeat(np.arange(m ** 3), npatch.ravel())
    origin = np.stack(np.unravel_index(cell_of_vertex, (m, m, m)), axis=-1).astype(np.float32)
    verts = (s / cnt[:, None]).astype(np.float32) + origin

    keys, quads = [], []
    idx = np.arange(n ** 3).reshape(n, n, n)
    for axis in range(3):
        b, c = (axis + 1) % 3, (axis + 2) % 3
        sl = [slice(None)] * 3
        sl[axis] = slice(0, n - 1)
        sl[b] = slice(1, n - 1)
        sl[c] = slice(1, n - 1)
        sl = tuple(sl)
        sh = [0, 0, 0]
        sh[axis] = 1
        v0 = g[sl]
        v1 = g[tuple(slice(s_.start + d, s_.stop + d) for s_, d in zip(sl, sh))]
        cross = np.isfinite(v0) & np.isfinite(v1) & ((v0 > 0) != (v1 > 0))
        pts = np.argwhere(cross) + np.array([s_.start for s_ in sl])
        q = np.zeros((len(pts), 4), dtype=np.int64)
        good = np.ones(len(pts), dtype=bool)
        for k, (db, dc) in enumerate(((-1, -1), (0, -1), (0, 0), (-1, 0))):
            cc = pts.copy()
            cc[:, b] += db
            cc[:, c] += dc
            cs = case[cc[:, 0], cc[:, 1], cc[:, 2]]
            good &= cs != 0
            bits = [0, 0, 0]
            bits[b], bits[c] = -db, -dc
            o0, o1 = (1, 2) if axis == 0 else ((0, 2) if axis == 1 else (0, 1))
            e = 4 * axis + bits[o0] + 2 * bits[o1]
            q[:, k] = voff[cc[:, 0], cc[:, 1], cc[:, 2]] + _PATCH[cs, e]
        inside0 = g[pts[:, 0], pts[:, 1], pts[:, 2]] > 0
        q[~inside0] = q[~inside0][:, [0, 3, 2, 1]]
        pts, q = pts[good], q[good]
        keys.append(idx[pts[:, 0], pts[:, 1], pts[:, 2]] * 3 + axis)
        quads.append(q)
    keys, quads = np.concatenate(keys), np.concatenate(quads)
    quads = quads[np.argsort(keys, kind="stable")]
    faces = np.stack([quads[:, [0, 1, 2]], quads[:, [0, 2, 3]]], axis=1).reshape(-1, 3)
    return verts, faces


def sha256(t: torch.Tensor) -> str:
    import hashlib

    return hashlib.sha256(t.detach().cpu().contiguous().numpy().tobytes()).hexdigest()


def mesh_stats(verts: np.ndarray, faces: np.ndarray):
    """-> (edges used by exactly 2 faces, Euler characteristic V - E + F over referenced vertices, signed volume)."""
    e = np.sort(np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]]), axis=1)
    _, counts = np.unique(e, axis=0, return_counts=True)
    nv = len(np.unique(faces))
    chi = nv - len(counts) + len(faces)
    v = verts.astype(np.float64)
    vol = np.einsum("ij,ij->i", v[faces[:, 0]], np.cross(v[faces[:, 1]], v[faces[:, 2]])).sum() / 6.0
    return bool((counts == 2).all()), chi, vol
