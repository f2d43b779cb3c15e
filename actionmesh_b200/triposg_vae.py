"""Stage 0's anchor mesh on the CUDA path: the decoder side of TripoSG's VAE and the octree + dual-marching-cubes extraction
that turn the denoised latent into the mesh Stage II deforms (SURVEY 8(f) row f2).

  B200TripoSGVAE.decode        TripoSGVAEModel.decode(z, sampled_points).sample   (autoencoder_kl_triposg.py:193-216,481-533)
  B200TripoSGVAE.extract_mesh  TripoSGPipelinePlus's default mesh path: flash_extract_geometry(latents, vae, bounds=±1.005,
                               octree_depth=9) (triposg/inference_utils.py:318-479) -> mesh with vertex normals

The decoder's 16 self-attention blocks and the query block's K/V do not depend on the query points, so they run ONCE per
latent (`prepare`); the reference recomputes them in every `vae.decode` call.  Precision: bf16 GEMM / attention operands with
fp32 accumulation, fp32 residual stream, LayerNorm statistics, coordinates and point embedding — the recipe and tolerance of
Stage 0's DiT.  (The reference runs this model in fp16, pipeline.py:140-142; the fp32 modules are the yardstick.)
There is no torch arithmetic on the path: torch allocates buffers and views them.
"""
from __future__ import annotations

import json
import math
import os
from dataclasses import dataclass, field
from typing import Callable, Optional

import numpy as np
import torch

from . import ops
from ._lib import AmbError
from .denoiser import repack_cross_kv, repack_self_qkv
from .pipeline import Mesh, _vertex_normals

DEFAULT_BOUNDS = (-1.005, -1.005, -1.005, 1.005, 1.005, 1.005)   # actionmesh/external/triposg.py:35-100
INVALID = -10000.0                                                 # flash_extract_geometry's "not queried" fill


@dataclass
class TripoSGVAEConfig:
    """Constructor arguments of TripoSGVAEModel (autoencoder_kl_triposg.py:221-233); the encoder's are accepted and unused."""
    in_channels: int = 3
    latent_channels: int = 64
    num_attention_heads: int = 8
    width_encoder: int = 512
    width_decoder: int = 1024
    num_layers_encoder: int = 8
    num_layers_decoder: int = 16
    embedding_type: str = "frequency"
    embed_frequency: int = 8
    embed_include_pi: bool = False

    @property
    def head_dim(self) -> int:
        return self.width_decoder // self.num_attention_heads

    @property
    def query_dim(self) -> int:
        return self.in_channels * (2 * self.embed_frequency + 1)


@dataclass
class AnchorMesh(Mesh):
    """`Mesh` plus the vertex normals Stage II reads (returned when trimesh is not installed)."""
    vertex_normals: "object" = field(default=None)


@dataclass
class LatentContext:
    """What `prepare` computes once per latent: the query block's keys and values, bf16 (N, H, d_h) views of one buffer."""
    kv: torch.Tensor
    k: torch.Tensor
    v: torch.Tensor


def octree_resolutions(octree_depth: int, min_resolution: int = 63, mini_grid_num: int = 4) -> list[int]:
    """The resolution ladder of inference_utils.py:333-344 ([63, 126, 252, 504] at depth 9)."""
    r = 2 ** octree_depth
    res = [r] if r < min_resolution else []
    while r >= min_resolution:
        res.append(r)
        r //= 2
    res.reverse()
    res[0] = round(res[0] / mini_grid_num) * mini_grid_num - 1
    for i in range(1, len(res)):
        res[i] = res[0] * 2 ** i
    return res


def refine_octree(query: Callable[[torch.Tensor], torch.Tensor], bounds=DEFAULT_BOUNDS, octree_depth: int = 9,
                  device="cuda") -> torch.Tensor:
    """flash_extract_geometry's refinement (inference_utils.py:333-460) up to the grid it hands to DiffDMC.

    `query(xyz)`: (P, 3) fp32 CUDA points -> fp32 logits (P, k) whose column 0 is used (any row stride).  Returns the final
    (n, n, n) fp32 grid, NaN where nothing was queried.  One host sync per finer level (the point count)."""
    dev = torch.device(device)
    lo = np.asarray(bounds[0:3], dtype=np.float64)
    hi = np.asarray(bounds[3:6], dtype=np.float64)
    size = hi - lo
    res = octree_resolutions(octree_depth)
    n = res[0] + 1
    axes = [np.linspace(lo[i], hi[i], n, dtype=np.float32) for i in range(3)]   # generate_dense_grid_points_2
    xyz = np.stack(np.meshgrid(*axes, indexing="ij"), axis=-1).reshape(-1, 3)
    grid = torch.empty(n, n, n, dtype=torch.float32, device=dev)
    ops.grid_scatter(query(torch.from_numpy(xyz).to(dev)), torch.arange(n ** 3, dtype=torch.int32, device=dev), grid)
    for r in res[1:]:
        last = r == res[-1]
        mask = ops.octree_near_surface(grid)
        if not last:
            mask = ops.octree_dilate(ops.octree_dilate(mask))
        fine = ops.octree_mark_upsampled(mask)
        for _ in range(2 if last else 1):
            fine = ops.octree_dilate(fine)
        del mask
        step = (size / r).astype(np.float32)                # torch.tensor(resolution, dtype=float32)
        pts, idx = ops.octree_points(fine, step, lo.astype(np.float32))
        del fine
        grid = ops.grid_fill(torch.empty(r + 1, r + 1, r + 1, dtype=torch.float32, device=dev), INVALID)
        if pts.shape[0]:
            ops.grid_scatter(query(pts), idx, grid)
    return ops.grid_replace(grid, INVALID, float("nan"))


def mesh_from_grid(grid: torch.Tensor, bounds=DEFAULT_BOUNDS, octree_depth: int = 9) -> tuple[np.ndarray, np.ndarray]:
    """Dual marching cubes of the refined grid and the reference's vertex scale (inference_utils.py:466-473) ->
    (vertices (V, 3) float32, faces (F, 3) int64), faces wound outward from the logits > 0 region.

    The scale divides by 2**octree_depth (512 at depth 9) although the grid spans 504 cells: the reference's mesh is 504/512
    of the box, and so is this one."""
    v, f = ops.dual_marching_cubes(grid)
    lo = np.asarray(bounds[0:3], dtype=np.float64)
    size = np.asarray(bounds[3:6], dtype=np.float64) - lo
    vertices = v.cpu().numpy() / (2 ** octree_depth) * size + lo
    return vertices.astype(np.float32), f.cpu().numpy().astype(np.int64)


def make_mesh(vertices: np.ndarray, faces: np.ndarray):
    """trimesh.Trimesh(v, f) as the reference returns (triposg.py), or the package's `AnchorMesh` with vertex normals."""
    try:
        import trimesh

        return trimesh.Trimesh(vertices, faces)
    except ImportError:
        vt = torch.from_numpy(vertices)
        n = _vertex_normals(vt, torch.from_numpy(faces)) if len(faces) else torch.zeros_like(vt)
        return AnchorMesh(vertices=vertices, faces=faces, vertex_normals=n.numpy())


class B200TripoSGVAE:
    """Decoder side of TripoSGVAEModel: same constructor arguments, state-dict keys (`post_quant.*`, `decoder.*`; the
    encoder's keys are ignored), `from_pretrained(f"{triposg_dir}/vae")` and `decode(z, sampled_points)`."""

    QUERY_CHUNK = 262144   # query rows per pass: ~4.6 GB of activations at width 1024

    def __init__(self, config: Optional[TripoSGVAEConfig] = None, **kwargs):
        self.config = config or TripoSGVAEConfig(**kwargs)
        c = self.config
        if c.embedding_type != "frequency":
            raise AmbError(f"embedding_type {c.embedding_type!r} is not supported")
        if c.head_dim != 128:
            raise AmbError(f"B200TripoSGVAE needs head_dim 128 (got {c.head_dim})")
        if c.width_decoder not in (256, 512, 1024, 2048, 4096):
            raise AmbError(f"unsupported width_decoder {c.width_decoder}")
        if c.in_channels != 3:
            raise AmbError("query points must be 3-D")
        self._device = torch.device("cpu")
        self._w: dict = {}
        self._loaded = False
        self._qpad = 64 * ((c.query_dim + 63) // 64)

    # ------------------------------------------------------------------ nn.Module-like surface
    @property
    def device(self) -> torch.device:
        return self._device

    def eval(self):
        return self

    def to(self, device):
        device = torch.device(device)
        if device.type != "cuda":
            raise AmbError("B200TripoSGVAE only runs on a CUDA (sm_90) device; there is no CPU path")
        if self._loaded and device != self._device:
            self._w = {k: v.to(device) for k, v in self._w.items()}
        self._device = device
        return self

    @classmethod
    def from_pretrained(cls, path: str, device="cuda") -> "B200TripoSGVAE":
        """Diffusers layout: `config.json` + `diffusion_pytorch_model.safetensors` (or `model.safetensors` / `.bin`)."""
        kwargs = {}
        cfg_path = os.path.join(path, "config.json")
        if os.path.exists(cfg_path):
            raw = json.load(open(cfg_path))
            kwargs = {k: v for k, v in raw.items() if k in TripoSGVAEConfig.__dataclass_fields__}
        model = cls(TripoSGVAEConfig(**kwargs)).to(device)
        for name in ("diffusion_pytorch_model.safetensors", "model.safetensors"):
            st = os.path.join(path, name)
            if os.path.exists(st):
                from safetensors.torch import load_file

                model.load_state_dict(load_file(st))
                return model
        model.load_state_dict(torch.load(os.path.join(path, "diffusion_pytorch_model.bin"), map_location="cpu"))
        return model

    @ops.on_device
    def load_state_dict(self, sd: dict) -> None:
        """Pack the weights: bf16 GEMM operands (self-attention QKV fused with the head split folded in, cross K/V likewise,
        proj_query K-padded to 64, proj_out N-padded to 64 and negated); biases and norm weights fp32."""
        c = self.config
        dev = self._device
        if dev.type != "cuda":
            raise AmbError("call .to('cuda') before load_state_dict")
        H, D, L = c.num_attention_heads, c.width_decoder, c.num_layers_decoder

        def f32(name):
            return sd[name].detach().to(device=dev, dtype=torch.float32).contiguous()

        def W(name):
            return f32(name).to(torch.bfloat16).contiguous()

        w = {"post_quant.w": W("post_quant.weight"), "post_quant.b": f32("post_quant.bias")}
        for i in range(L + 1):
            p, q = f"decoder.blocks.{i}.", f"b{i}."
            norm_attn, attn = ("norm2", "attn2") if i == L else ("norm1", "attn1")
            for src, dst in ((norm_attn, "norm_attn"), ("norm3", "norm_ff")):
                w[q + dst + ".g"], w[q + dst + ".b"] = f32(p + src + ".weight"), f32(p + src + ".bias")
            wq, wk, wv = (f32(p + f"{attn}.to_{n}.weight") for n in "qkv")
            if i < L:
                w[q + "qkv"] = repack_self_qkv(wq, wk, wv, H).to(torch.bfloat16).contiguous()
            else:
                w[q + "q"] = wq.to(torch.bfloat16).contiguous()
                w[q + "kv"] = repack_cross_kv(wk, wv, H).to(torch.bfloat16).contiguous()
                w[q + "norm_cross.g"], w[q + "norm_cross.b"] = f32(p + "attn2.norm_cross.weight"), f32(p + "attn2.norm_cross.bias")
            w[q + "o.w"], w[q + "o.b"] = W(p + f"{attn}.to_out.0.weight"), f32(p + f"{attn}.to_out.0.bias")
            w[q + "ff1.w"], w[q + "ff1.b"] = W(p + "ff.net.0.proj.weight"), f32(p + "ff.net.0.proj.bias")
            w[q + "ff2.w"], w[q + "ff2.b"] = W(p + "ff.net.2.weight"), f32(p + "ff.net.2.bias")
        pq = torch.zeros(D, self._qpad, dtype=torch.float32, device=dev)
        pq[:, :c.query_dim].copy_(f32("decoder.proj_query.weight"))
        w["proj_query.w"], w["proj_query.b"] = pq.to(torch.bfloat16), f32("decoder.proj_query.bias")
        w["norm_out.g"], w["norm_out.b"] = f32("decoder.norm_out.weight"), f32("decoder.norm_out.bias")
        # proj_out (1 x D) padded to 64 output columns; TripoSGDecoder.forward's `logits * -1` folded in (exact in bf16/fp32)
        po = torch.zeros(64, D, dtype=torch.float32, device=dev)
        po[:1].copy_(f32("decoder.proj_out.weight"))
        pb = torch.zeros(64, dtype=torch.float32, device=dev)
        pb[:1].copy_(f32("decoder.proj_out.bias"))
        w["proj_out.w"], w["proj_out.b"] = po.neg().to(torch.bfloat16), pb.neg()
        self._w = w
        self._loaded = True

    @ops.on_device
    def init_random_(self, seed: int = 1237) -> None:
        """Synthetic weights for benchmarks (no checkpoints offline), generated on the GPU like B200Autoencoder's."""
        c = self.config
        dev = self._device
        g = torch.Generator(device=dev).manual_seed(seed)
        D, L = c.width_decoder, c.num_layers_decoder
        rs = 1.0 / math.sqrt(L + 1)

        def lin(name, out_f, in_f, scale=1.0, bias=True):
            bound = 1.0 / math.sqrt(in_f)
            sd[name + ".weight"] = (torch.rand(out_f, in_f, generator=g, device=dev) * 2 - 1) * bound * scale
            if bias:
                sd[name + ".bias"] = (torch.rand(out_f, generator=g, device=dev) * 2 - 1) * bound * scale

        def ln(name):
            sd[name + ".weight"], sd[name + ".bias"] = torch.ones(D, device=dev), torch.zeros(D, device=dev)

        sd = {}
        lin("post_quant", D, c.latent_channels)
        lin("decoder.proj_query", D, c.query_dim)
        lin("decoder.proj_out", 1, D)
        ln("decoder.norm_out")
        for i in range(L + 1):
            p = f"decoder.blocks.{i}."
            a = "attn2" if i == L else "attn1"
            ln(p + ("norm2" if i == L else "norm1"))
            ln(p + "norm3")
            if i == L:
                ln(p + "attn2.norm_cross")
            for n in ("to_q", "to_k", "to_v"):
                lin(p + f"{a}.{n}", D, D, bias=False)
            lin(p + f"{a}.to_out.0", D, D, scale=rs)
            lin(p + "ff.net.0.proj", 4 * D, D)
            lin(p + "ff.net.2", D, 4 * D, scale=rs)
        self.load_state_dict(sd)

    # ------------------------------------------------------------------ decode
    @ops.on_device
    @torch.no_grad()
    def prepare(self, z: torch.Tensor) -> LatentContext:
        """One latent (N, C) -> the query block's K/V: post_quant, the 16 self-attention blocks (fp32 residual stream), then
        norm_cross and the fused K/V GEMM (autoencoder_kl_triposg.py:199-203,491; attention_processor.py:232-262)."""
        if not self._loaded:
            raise AmbError("B200TripoSGVAE: weights not loaded")
        c, w, dev = self.config, self._w, self._device
        N = z.shape[0]
        D, H, dh, L = c.width_decoder, c.num_attention_heads, c.head_dim, c.num_layers_decoder
        bf, f32 = torch.bfloat16, torch.float32
        E = lambda *s, dtype=bf: torch.empty(*s, dtype=dtype, device=dev)
        h, xn, qkv, att, ff = E(N, D, dtype=f32), E(N, D), E(N, 3 * D), E(N, D), E(N, 4 * D)
        zb = ops.cast_bf16(z.detach().to(device=dev, dtype=f32).contiguous())
        ops.gemm(zb, w["post_quant.w"], h, bias=w["post_quant.b"], tag="vae_trunk")
        scale = 1.0 / math.sqrt(dh)
        for i in range(L):
            q = f"b{i}."
            ops.layernorm(h, w[q + "norm_attn.g"], w[q + "norm_attn.b"], 1e-5, out=xn)
            ops.gemm(xn, w[q + "qkv"], qkv, tag="vae_trunk")
            ops.flash_attn(qkv[:, 0:D].view(1, N, H, dh), qkv[:, D:2 * D].view(1, N, H, dh), qkv[:, 2 * D:].view(1, N, H, dh),
                           att.view(1, N, H, dh), scale, tag="vae_trunk_attn")
            ops.gemm(att, w[q + "o.w"], h, bias=w[q + "o.b"], residual=h, tag="vae_trunk")
            ops.layernorm(h, w[q + "norm_ff.g"], w[q + "norm_ff.b"], 1e-5, out=xn)
            ops.gemm(xn, w[q + "ff1.w"], ff, bias=w[q + "ff1.b"], act=1, tag="vae_trunk")
            ops.gemm(ff, w[q + "ff2.w"], h, bias=w[q + "ff2.b"], residual=h, tag="vae_trunk")
        q = f"b{L}."
        ops.layernorm(h, w[q + "norm_cross.g"], w[q + "norm_cross.b"], 1e-5, out=xn)
        kv = ops.gemm(xn, w[q + "kv"], E(N, 2 * D), tag="vae_trunk")          # [K(h,d) | V(h,d)]
        return LatentContext(kv=kv, k=kv[:, :D].view(1, N, H, dh), v=kv[:, D:].view(1, N, H, dh))

    @ops.on_device
    @torch.no_grad()
    def query(self, ctx: LatentContext, points: torch.Tensor, chunk: Optional[int] = None) -> torch.Tensor:
        """(P, 3) fp32 points -> (P, 64) fp32 whose column 0 is the logit (the other columns are zero padding)."""
        c, w, dev = self.config, self._w, self._device
        P = points.shape[0]
        D, H, dh = c.width_decoder, c.num_attention_heads, c.head_dim
        q = f"b{c.num_layers_decoder}."
        bf, f32 = torch.bfloat16, torch.float32
        out = torch.empty(P, 64, dtype=f32, device=dev)
        rows = min(P, chunk or self.QUERY_CHUNK)
        if rows == 0:
            return out
        E = lambda *s, dtype=bf: torch.empty(*s, dtype=dtype, device=dev)
        eb, x, xn, qb, att, ff = E(rows, self._qpad), E(rows, D, dtype=f32), E(rows, D), E(rows, D), E(rows, D), E(rows, 4 * D)
        pts = points.detach().to(device=dev, dtype=f32).contiguous()
        scale = 1.0 / math.sqrt(dh)
        Sk = ctx.kv.shape[0]
        for r0 in range(0, P, rows):
            m = min(rows, P - r0)
            e32 = ops.point_embedding(pts[r0:r0 + m], c.embed_frequency, c.embed_include_pi, self._qpad)
            ops.cast_bf16(e32, eb[:m])
            ops.gemm(eb[:m], w["proj_query.w"], x[:m], bias=w["proj_query.b"], tag="vae_query")
            ops.layernorm(x[:m], w[q + "norm_attn.g"], w[q + "norm_attn.b"], 1e-5, out=xn[:m])
            ops.gemm(xn[:m], w[q + "q"], qb[:m], tag="vae_query")
            ops.flash_attn(qb[:m].view(1, m, H, dh), ctx.k.view(1, Sk, H, dh), ctx.v.view(1, Sk, H, dh),
                           att[:m].view(1, m, H, dh), scale, tag="vae_query_attn")
            ops.gemm(att[:m], w[q + "o.w"], x[:m], bias=w[q + "o.b"], residual=x[:m], tag="vae_query")
            ops.layernorm(x[:m], w[q + "norm_ff.g"], w[q + "norm_ff.b"], 1e-5, out=xn[:m])
            ops.gemm(xn[:m], w[q + "ff1.w"], ff[:m], bias=w[q + "ff1.b"], act=1, tag="vae_query")
            ops.gemm(ff[:m], w[q + "ff2.w"], x[:m], bias=w[q + "ff2.b"], residual=x[:m], tag="vae_query")
            ops.layernorm(x[:m], w["norm_out.g"], w["norm_out.b"], 1e-5, out=xn[:m])
            ops.gemm(xn[:m], w["proj_out.w"], out[r0:r0 + m], bias=w["proj_out.b"], tag="vae_query")
        return out

    @torch.no_grad()
    def decode(self, z: torch.Tensor, sampled_points: torch.Tensor, return_dict: bool = True):
        """TripoSGVAEModel.decode: (B, N, C) latents, (B, P, 3) points -> (B, P, 1) fp32 logits (`.sample` of the reference's
        DecoderOutput; returned as the tensor itself, or a 1-tuple with return_dict=False)."""
        B, P = sampled_points.shape[:2]
        out = torch.empty(B, P, 1, dtype=torch.float32, device=self._device)
        for b in range(B):
            logits = self.query(self.prepare(z[b]), sampled_points[b].reshape(P, 3))
            out[b, :, 0].copy_(logits[:, 0])
        return out if return_dict else (out,)

    # ------------------------------------------------------------------ mesh
    @torch.no_grad()
    def extract_geometry(self, latents: torch.Tensor, bounds=DEFAULT_BOUNDS, octree_depth: int = 9,
                         decode: Optional[Callable] = None) -> list:
        """flash_extract_geometry(latents, vae, bounds, octree_depth) -> [(vertices, faces)] per latent of the batch.
        `decode(xyz) -> (P, k) logits` replaces the decoder (e.g. an analytic field); default: this VAE."""
        out = []
        for b in range(latents.shape[0]):
            if decode is None:
                ctx = self.prepare(latents[b])
                fn = lambda xyz, ctx=ctx: self.query(ctx, xyz)
            else:
                fn = decode
            with torch.cuda.device(self._device):
                grid = refine_octree(fn, bounds, octree_depth, self._device)
                out.append(mesh_from_grid(grid, bounds, octree_depth))
            del grid
        return out

    def extract_mesh(self, latents: torch.Tensor, bounds=DEFAULT_BOUNDS, octree_depth: int = 9):
        """`mesh_extractor` of TripoSGStage0: (1, N, C) latents -> mesh with .vertices, .faces, .vertex_normals."""
        v, f = self.extract_geometry(latents, bounds, octree_depth)[0]
        return make_mesh(v, f)
