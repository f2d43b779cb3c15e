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

The encoder side (`encode`, `encode_to_latent`) turns the surface samples of a user-supplied mesh into the anchor latent of
the {video + 3D mesh} -> 4D pipeline: farthest-point sampling on the GPU (csrc/point_sampling.cu), then TripoSGEncoder (one
cross-attention block from the sampled points to all surface points, then self-attention blocks) and `quant` on the same
kernels, and the posterior sample in one elementwise kernel.  Coordinates, point embedding and FPS stay fp32; the reference
rounds the surface to fp16 before embedding it (pipeline_with_3d.py:97-105) and runs the VAE in fp16.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Callable, Optional

import numpy as np
import torch

from . import blocks, ops
from ._lib import AmbError
from .blocks import TRIPOSG_BLOCK_KEYS, SyntheticWeights, V, W, pack_block, remap_triposg_state_dict
from .module import B200Module
from .pipeline import Mesh, _vertex_normals

DEFAULT_BOUNDS = (-1.005, -1.005, -1.005, 1.005, 1.005, 1.005)   # actionmesh/external/triposg.py:35-100
INVALID = -10000.0                                                 # flash_extract_geometry's "not queried" fill


@dataclass
class TripoSGVAEConfig:
    """Constructor arguments of TripoSGVAEModel (autoencoder_kl_triposg.py:221-233)."""
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

    @property
    def encoder_head_dim(self) -> int:
        return self.width_encoder // self.num_attention_heads

    @property
    def encoder_in_dim(self) -> int:
        """[embed(xyz) | normal]: the encoder's proj_in input (autoencoder_kl_triposg.py:250-252,442-451)."""
        return self.query_dim + self.in_channels

    def encoder_supported(self) -> Optional[str]:
        """None when the encoder side runs on this build, else the reason it does not."""
        if self.encoder_head_dim not in (64, 128) or self.encoder_head_dim * self.num_attention_heads != self.width_encoder:
            return f"the encoder needs head_dim 64 or 128 (got width_encoder {self.width_encoder} / {self.num_attention_heads} heads)"
        if self.width_encoder not in (256, 512, 1024, 2048, 4096):
            return f"unsupported width_encoder {self.width_encoder}"
        return None


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


class DiagonalGaussianDistribution:
    """The posterior of vae.py:8-36 over fp32 `parameters` (..., 2C) = [mean | logvar] (the `quant` output, read in place):
    `mean` is a view, `logvar` (clamped to [-30, 20]) and `std` = exp(0.5 logvar) come from one kernel, and
    `sample(generator)` = mean + std * eps with eps ~ torch.randn from `generator` (on the generator's device)."""

    def __init__(self, parameters: torch.Tensor):
        C = parameters.shape[-1] // 2
        self.parameters = parameters
        self._rows = parameters.reshape(-1, 2 * C)
        self.mean = parameters[..., :C]
        self.logvar = torch.empty(self.mean.shape, dtype=torch.float32, device=parameters.device)
        self.std = torch.empty_like(self.logvar)
        ops.gaussian_sample(self._rows, logvar=self.logvar.view(-1, C), std=self.std.view(-1, C))

    @torch.no_grad()
    def sample(self, generator: Optional[torch.Generator] = None, eps: Optional[torch.Tensor] = None) -> torch.Tensor:
        """mean + std * eps; `eps` (same shape as mean) replaces the draw when given."""
        dev = self.parameters.device
        if eps is None:
            gdev = generator.device if generator is not None else dev
            eps = torch.randn(self.mean.shape, generator=generator, device=gdev, dtype=torch.float32)
        eps = eps.to(device=dev, dtype=torch.float32).contiguous()
        z = torch.empty(self.mean.shape, dtype=torch.float32, device=dev)
        ops.gaussian_sample(self._rows, eps.view(-1, self.mean.shape[-1]), z=z.view(-1, self.mean.shape[-1]))
        return z

    def mode(self) -> torch.Tensor:
        return self.mean


@dataclass
class EncoderOutput:
    """diffusers' AutoencoderKLOutput: the posterior of `B200TripoSGVAE.encode`."""
    latent_dist: DiagonalGaussianDistribution


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


class B200TripoSGVAE(B200Module):
    """TripoSGVAEModel on the CUDA path: same constructor arguments, state-dict keys (`post_quant.*`, `decoder.*`, and the
    encoder side's `encoder.*`, `quant.*` when present), `from_pretrained(f"{triposg_dir}/vae")`, `decode(z, sampled_points)`
    and, for a user-supplied mesh, `encode(surface)` / `encode_to_latent(surface)` (actionmesh/external/triposg.py:103-172)."""

    config_class = TripoSGVAEConfig
    weight_files = ("diffusion_pytorch_model.safetensors", "model.safetensors", "diffusion_pytorch_model.bin")
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
        super().__init__()
        self._has_encoder = False
        self._qpad = 64 * ((c.query_dim + 63) // 64)
        self._epad = 64 * ((c.encoder_in_dim + 63) // 64)

    def _pack_state_dict(self, sd: dict, dev: torch.device) -> dict:
        """Pack the weights: bf16 GEMM operands (self-attention QKV fused with the head split folded in, cross K/V likewise,
        proj_query K-padded to 64, proj_out N-padded to 64 and negated); biases and norm weights fp32.  The encoder side
        (`encoder.*`, `quant.*`: proj_in K-padded 54 -> 64) is packed too when the dict has it.  The DiT blocks go through
        the TripoSG -> ActionMesh key map and are packed under `b{i}.` (decoder) and `e{i}.` (encoder)."""
        c = self.config
        H, D, L = c.num_attention_heads, c.width_decoder, c.num_layers_decoder
        f32 = lambda name: V(sd[name], dev)
        w = {"post_quant.w": W(sd["post_quant.weight"], dev), "post_quant.b": f32("post_quant.bias")}
        blk = remap_triposg_state_dict(remap_triposg_state_dict(sd, "decoder.blocks."), "encoder.blocks.")
        for i in range(L + 1):
            pack_block(w, blk, f"decoder.blocks.{i}.", f"b{i}.", H, dev)
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
        self._has_encoder = "quant.weight" in sd
        if self._has_encoder:
            why = c.encoder_supported()
            if why is not None:
                raise AmbError(f"B200TripoSGVAE: {why}")
            # block 0 cross-attends from the sampled points to all surface points; blocks 1..L are self-attention
            for i in range(c.num_layers_encoder + 1):
                pack_block(w, blk, f"encoder.blocks.{i}.", f"e{i}.", H, dev)
            pi = torch.zeros(c.width_encoder, self._epad, dtype=torch.float32, device=dev)
            pi[:, :c.encoder_in_dim].copy_(f32("encoder.proj_in.weight"))
            w["proj_in.w"], w["proj_in.b"] = pi.to(torch.bfloat16), f32("encoder.proj_in.bias")
            w["enc_norm_out.g"], w["enc_norm_out.b"] = f32("encoder.norm_out.weight"), f32("encoder.norm_out.bias")
            w["quant.w"], w["quant.b"] = W(sd["quant.weight"], dev), f32("quant.bias")
        return w

    @ops.on_device
    def init_random_(self, seed: int = 1237) -> None:
        """Synthetic weights for benchmarks (no checkpoints offline), generated on the GPU like B200Autoencoder's."""
        c = self.config
        D, L = c.width_decoder, c.num_layers_decoder
        sd = SyntheticWeights(seed, self._device)
        sd.linear("post_quant", D, c.latent_channels)
        sd.linear("decoder.proj_query", D, c.query_dim)
        sd.linear("decoder.proj_out", 1, D)
        sd.layernorm("decoder.norm_out", D)
        for i in range(L + 1):
            sd.dit_block(f"decoder.blocks.{i}.", D, 4 * D, 1.0 / math.sqrt(L + 1), ("x_attn" if i == L else "s_attn",),
                         norm_cross=i == L)
        if c.encoder_supported() is None:
            # encoder from its own generator, so the decoder's weights are the same with or without it
            We, Le = c.width_encoder, c.num_layers_encoder
            enc = SyntheticWeights(seed + 1, self._device)
            enc.linear("encoder.proj_in", We, c.encoder_in_dim)
            enc.linear("quant", 2 * c.latent_channels, We)
            enc.layernorm("encoder.norm_out", We)
            for i in range(Le + 1):
                enc.dit_block(f"encoder.blocks.{i}.", We, 4 * We, 1.0 / math.sqrt(Le + 1), ("x_attn" if i == 0 else "s_attn",),
                              norm_cross=i == 0)
            sd.update(enc)
        to_triposg = [(b, a) for a, b in TRIPOSG_BLOCK_KEYS]
        sd = blocks.remap_block_keys(blocks.remap_block_keys(sd, to_triposg, "decoder.blocks."), to_triposg, "encoder.blocks.")
        self.load_state_dict(sd)

    # ------------------------------------------------------------------ decode
    @ops.on_device
    @torch.no_grad()
    def prepare(self, z: torch.Tensor) -> LatentContext:
        """One latent (N, C) -> the query block's K/V: post_quant, the 16 self-attention blocks (fp32 residual stream), then
        norm_cross and the fused K/V GEMM (autoencoder_kl_triposg.py:199-203,491; attention_processor.py:232-262)."""
        self._check_loaded()
        c, w, dev = self.config, self._w, self._device
        N = z.shape[0]
        D, H, dh, L = c.width_decoder, c.num_attention_heads, c.head_dim, c.num_layers_decoder
        bf, f32 = torch.bfloat16, torch.float32
        E = lambda *s, dtype=bf: torch.empty(*s, dtype=dtype, device=dev)
        h, xn, qkv, att, ff = E(N, D, dtype=f32), E(N, D), E(N, 3 * D), E(N, D), E(N, 4 * D)
        zb = ops.cast_bf16(z.detach().to(device=dev, dtype=f32).contiguous())
        ops.gemm(zb, w["post_quant.w"], h, bias=w["post_quant.b"], tag="vae_trunk")
        for i in range(L):
            blocks.attention_half(w, f"b{i}.", h, xn, qkv, att, (1, N), H, tag="vae_trunk", attn_tag="vae_trunk_attn")
            blocks.output_half(w, f"b{i}.", "s", h, att, xn, ff, tag="vae_trunk")
        q = f"b{L}."
        ops.layernorm(h, w[q + "norm_cross.g"], w[q + "norm_cross.b"], 1e-5, out=xn)
        kv = ops.gemm(xn, w[q + "x.kv"], E(N, 2 * D), tag="vae_trunk")          # [K(h,d) | V(h,d)]
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
            ops.layernorm(x[:m], w[q + "norm_x_attn.g"], w[q + "norm_x_attn.b"], 1e-5, out=xn[:m])
            ops.gemm(xn[:m], w[q + "x.q"], qb[:m], tag="vae_query")
            ops.flash_attn(qb[:m].view(1, m, H, dh), ctx.k.view(1, Sk, H, dh), ctx.v.view(1, Sk, H, dh),
                           att[:m].view(1, m, H, dh), scale, tag="vae_query_attn")
            blocks.output_half(w, q, "x", x[:m], att[:m], xn[:m], ff[:m], tag="vae_query")
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

    # ------------------------------------------------------------------ encode
    @ops.on_device
    @torch.no_grad()
    def encode_points(self, x_kv: torch.Tensor, x_q: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """TripoSGEncoder + quant for one shape (autoencoder_kl_triposg.py:26-87,439-457): all surface points x_kv (N, 6) and
        the sampled points x_q (T, 6), fp32 [xyz | normal] rows -> (T, 2 * latent_channels) fp32 `quant` output."""
        if not self._loaded or not self._has_encoder:
            raise AmbError("B200TripoSGVAE: encoder weights not loaded")
        c, w, dev = self.config, self._w, self._device
        N, T = x_kv.shape[0], x_q.shape[0]
        D, H, dh, L = c.width_encoder, c.num_attention_heads, c.encoder_head_dim, c.num_layers_encoder
        bf, f32 = torch.bfloat16, torch.float32
        E = lambda *s, dtype=bf: torch.empty(*s, dtype=dtype, device=dev)
        if out is None:
            out = E(T, 2 * c.latent_channels, dtype=f32)
        h, xn, qkv, att, ff = E(T, D, dtype=f32), E(T, D), E(T, 3 * D), E(T, D), E(T, 4 * D)
        ctx, ctxn = E(N, D, dtype=f32), E(N, D)
        F, pi = c.embed_frequency, c.embed_include_pi
        # x_kv = [embed(xyz) | normal] of every surface point, x_q the same of the sampled points; one shared proj_in
        ekv = ops.cast_bf16(ops.point_embedding(x_kv.detach().to(device=dev, dtype=f32).contiguous(), F, pi, self._epad))
        eq = ops.cast_bf16(ops.point_embedding(x_q.detach().to(device=dev, dtype=f32).contiguous(), F, pi, self._epad))
        ops.gemm(eq, w["proj_in.w"], h, bias=w["proj_in.b"], tag="vae_encoder")
        ops.gemm(ekv, w["proj_in.w"], ctx, bias=w["proj_in.b"], tag="vae_encoder")
        del ekv, eq
        # block 0: cross-attention to the norm_cross'ed surface tokens
        q = "e0."
        ops.layernorm(ctx, w[q + "norm_cross.g"], w[q + "norm_cross.b"], 1e-5, out=ctxn)
        kv = ops.gemm(ctxn, w[q + "x.kv"], E(N, 2 * D), tag="vae_encoder")          # [K(h,d) | V(h,d)]
        del ctx, ctxn
        ops.layernorm(h, w[q + "norm_x_attn.g"], w[q + "norm_x_attn.b"], 1e-5, out=xn)
        qb = ops.gemm(xn, w[q + "x.q"], E(T, D), tag="vae_encoder")
        ops.flash_attn(qb.view(1, T, H, dh), kv[:, :D].view(1, N, H, dh), kv[:, D:].view(1, N, H, dh), att.view(1, T, H, dh),
                       1.0 / math.sqrt(dh), tag="vae_encoder_attn")
        del qb, kv
        blocks.output_half(w, q, "x", h, att, xn, ff, tag="vae_encoder")
        for i in range(1, L + 1):
            blocks.attention_half(w, f"e{i}.", h, xn, qkv, att, (1, T), H, tag="vae_encoder", attn_tag="vae_encoder_attn")
            blocks.output_half(w, f"e{i}.", "s", h, att, xn, ff, tag="vae_encoder")
        ops.layernorm(h, w["enc_norm_out.g"], w["enc_norm_out.b"], 1e-5, out=xn)
        ops.gemm(xn, w["quant.w"], out, bias=w["quant.b"], tag="vae_encoder")
        return out

    @ops.on_device
    @torch.no_grad()
    def sample_features(self, x: torch.Tensor, num_tokens: int = 2048, seed: Optional[int] = None,
                        generator: Optional[torch.Generator] = None) -> tuple[torch.Tensor, torch.Tensor]:
        """TripoSGVAE._sample_features (actionmesh/external/triposg.py:113-151): (B, N, 6) fp32 CUDA surface -> (the sampled
        rows (B, num_tokens, 6), their indices into the 4 * num_tokens subset (B, num_tokens) int64).

        The subset is `np.random.default_rng(seed).choice(N, 4 * num_tokens, replace=4 * num_tokens > N)` on the host, the
        reference's exact call; farthest-point sampling then runs on the GPU from `torch.randint(high=4 * num_tokens,
        size=(1,), generator=generator)` per batch element."""
        B, N = x.shape[:2]
        m = 4 * num_tokens
        if m > ops.FPS_MAX_POINTS:
            raise AmbError(f"num_tokens {num_tokens}: farthest-point sampling supports 4 * num_tokens <= {ops.FPS_MAX_POINTS}")
        subset = np.random.default_rng(seed).choice(N, m, replace=m > N)
        selected = x[:, torch.from_numpy(subset).to(x.device)]                       # (B, m, 6), a gather
        gdev = generator.device if generator is not None else torch.device("cpu")
        start = torch.cat([torch.randint(high=m, size=(1,), generator=generator, device=gdev) for _ in range(B)])
        idx = ops.farthest_point_sample(selected, num_tokens, start)
        return selected[torch.arange(B, device=x.device)[:, None], idx], idx

    @ops.on_device
    @torch.no_grad()
    def encode(self, x: torch.Tensor, return_dict: bool = True, num_tokens: int = 2048, seed: Optional[int] = None,
               generator: Optional[torch.Generator] = None):
        """TripoSGVAEModel.encode with TripoSGVAE's sampling (autoencoder_kl_triposg.py:439-479, external/triposg.py:113-151):
        (B, N, 6) surface [xyz | normal] -> `.latent_dist`, a `DiagonalGaussianDistribution` of (B, num_tokens, C).
        `seed` fixes the host subset, `generator` the FPS start (and is the natural one to pass to `.sample`)."""
        x = x.detach().to(device=self._device, dtype=torch.float32).contiguous()
        sampled, _ = self.sample_features(x, num_tokens, seed, generator)
        params = torch.empty(x.shape[0], num_tokens, 2 * self.config.latent_channels, dtype=torch.float32, device=self._device)
        for b in range(x.shape[0]):
            self.encode_points(x[b], sampled[b], out=params[b])
        posterior = DiagonalGaussianDistribution(params)
        return EncoderOutput(latent_dist=posterior) if return_dict else (posterior,)

    @torch.no_grad()
    def encode_to_latent(self, surface: torch.Tensor, seed: Optional[int] = None,
                         generator: Optional[torch.Generator] = None) -> torch.Tensor:
        """TripoSGVAE.encode_to_latent (external/triposg.py:153-172): (B, N, 6) surface -> posterior sample (B, 2048, C) fp32.
        With both `seed` and `generator` given the result is reproducible (the reference passes neither)."""
        return self.encode(surface, seed=seed, generator=generator).latent_dist.sample(generator)

    # ------------------------------------------------------------------ mesh
    @ops.on_device
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
            grid = refine_octree(fn, bounds, octree_depth, self._device)
            out.append(mesh_from_grid(grid, bounds, octree_depth))
            del grid
        return out

    def extract_mesh(self, latents: torch.Tensor, bounds=DEFAULT_BOUNDS, octree_depth: int = 9):
        """`mesh_extractor` of TripoSGStage0: (1, N, C) latents -> mesh with .vertices, .faces, .vertex_normals."""
        v, f = self.extract_geometry(latents, bounds, octree_depth)[0]
        return make_mesh(v, f)
