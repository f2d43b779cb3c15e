"""H100-native Stage-II temporal autoencoder — drop-in for `ActionMeshAutoencoder`
(actionmesh/model/temporal_autoencoder.py:30-269), the first "next" row of SURVEY 8(f).

Same duck type the pipeline uses (pipeline.py:186-199,358-372): `forward(latent, framestep, source_alpha, target_alphas,
query, step_callback) -> displacement (B, T_out, V, 3)`, `apply_displacement`, `.device / .eval() / .to() /
from_pretrained()`, the reference's state-dict keys.

Two precision regimes, as in the reference:
  * the 16-block self-attention trunk over the T*(N+1) latent+alpha tokens runs under autocast in the reference with an
    fp32 residual stream (`cat([bf16 latents, fp32 alpha])` promotes, temporal_autoencoder.py:256) and bf16 GEMMs/SDPA.
    Here: h fp32, LayerNorm fp32 -> bf16, fused QKV GEMM (head split folded in the weights, RoPE in the epilogue, no
    q/k norm), the wgmma flash attention, to_out/FF GEMMs with fp32 residual epilogues.  Tokens are laid out
    frame-major [N latents | 1 alpha token] per frame instead of the reference's [T*N latents | T alpha tokens]; every
    op of the block is token-local or permutation invariant (unmasked attention), and a token's RoPE position is its
    frame in both layouts, so results are identical and the denoiser's kernels are reused unchanged.
  * the final vertex-query cross-attention block runs with autocast DISABLED (fp32) in the reference
    (temporal_autoencoder.py:264-266).  Here it runs on the bf16 tensor cores at fp32-grade accuracy: every operand is
    split x = hi + lo and concatenated along K (ops.split3), attention is evaluated unfused per head as
    S = Q'K'^T (fp32) -> row softmax (fp32, ops.softmax_split3) -> O = P'V'^T, all with fp32 accumulation.
There is no torch arithmetic on the path (torch owns buffers and does two memcpy-style `copy_`s) and no CPU fallback.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Callable, Optional

import torch

from . import ops
from . import blocks
from ._lib import AmbError
from .blocks import SyntheticWeights, V, W, pack_block, repack_cross_kv
from .module import B200Module


@dataclass
class AutoencoderConfig:
    """Defaults of temporal_autoencoder.py:38-57."""
    in_channels: int = 3
    in_extra_channels: int = 3
    out_dim: int = 3
    latent_channels: int = 64
    width: int = 1024
    num_layers: int = 16
    num_attention_heads: int = 8
    embed_frequency: int = 8
    embed_include_pi: bool = False
    prediction_mode: str = "direct"
    temporal_context_size: int = 16

    @property
    def head_dim(self) -> int:
        return self.width // self.num_attention_heads

    @property
    def query_dim(self) -> int:
        return self.in_channels * (2 * self.embed_frequency + 1) + self.in_extra_channels


def _pad64(n: int) -> int:
    return (n + 63) // 64 * 64


class B200Autoencoder(B200Module):
    config_class = AutoencoderConfig
    QUERY_CHUNK = 16384  # vertex rows per score-matrix chunk (S chunk = 16384 x 32832 fp32 = 2.2 GB at the default shape)

    def __init__(self, config: Optional[AutoencoderConfig] = None, **kwargs):
        self.config = config or AutoencoderConfig(**kwargs)
        c = self.config
        if c.head_dim != 128:
            raise AmbError(f"B200Autoencoder needs head_dim 128 (got {c.head_dim})")
        if c.width not in (256, 512, 1024, 2048, 4096):
            raise AmbError(f"unsupported width {c.width}")
        if c.in_channels != 3:
            raise AmbError("query points must be 3-D")
        super().__init__()
        self.verbose = False
        self.prediction_mode = c.prediction_mode

    def _pack_state_dict(self, sd: dict, dev: torch.device) -> dict:
        """Pack the reference's state dict: trunk GEMM weights bf16 (QKV fused + head-permuted); the fp32 query-path
        weights as split-bf16 [hi | hi | lo] operands; biases / norm weights fp32."""
        c = self.config
        H, D = c.num_attention_heads, c.width

        def S3(t: torch.Tensor, kpad: Optional[int] = None, npad: Optional[int] = None) -> torch.Tensor:
            """fp32 (n, k) weight -> bf16 (npad, 3*kpad) [hi | hi | lo] via the split kernel."""
            n, k = t.shape
            kp, np_ = kpad or k, npad or n
            src = torch.zeros(np_, kp, dtype=torch.float32, device=dev)
            src[:n, :k].copy_(t)
            return ops.split3(src, torch.empty(np_, 3 * kp, dtype=torch.bfloat16, device=dev), weight=True)

        f32 = lambda name: V(sd[name], dev)
        w = {}
        w["post_quant.w"], w["post_quant.b"] = W(sd["post_quant.weight"], dev), f32("post_quant.bias")
        for i in range(c.num_layers):
            pack_block(w, sd, f"blocks.{i}.", f"blocks.{i}.", H, dev)
        # ---- fp32-grade query path (temporal_autoencoder.py:143-161)
        p = f"blocks.{c.num_layers}."
        self._qpad = _pad64(c.query_dim)
        w["proj_query.w3"], w["proj_query.b"] = S3(f32("proj_query.weight"), kpad=self._qpad), f32("proj_query.bias")
        for n in ("norm_x_attn", "norm_ff"):
            w[p + n + ".g"], w[p + n + ".b"] = f32(p + n + ".weight"), f32(p + n + ".bias")
        w[p + "norm_cross.g"], w[p + "norm_cross.b"] = f32(p + "x_attn.norm_cross.weight"), f32(p + "x_attn.norm_cross.bias")
        w[p + "x.q3"] = S3(f32(p + "x_attn.to_q.weight"))
        kv = repack_cross_kv(f32(p + "x_attn.to_k.weight"), f32(p + "x_attn.to_v.weight"), H)  # rows [K(h,d) | V(h,d)]
        w[p + "x.k3"] = S3(kv[:D].contiguous())
        w[p + "x.v3"] = S3(kv[D:].contiguous())  # used as the A operand of V^T = W_v ctx^T (weight split on both sides is symmetric)
        w[p + "x.o3"], w[p + "x.o.b"] = S3(f32(p + "x_attn.to_out.0.weight")), f32(p + "x_attn.to_out.0.bias")
        w[p + "ff1.w3"], w[p + "ff1.b"] = S3(f32(p + "ff.net.0.proj.weight")), f32(p + "ff.net.0.proj.bias")
        w[p + "ff2.w3"], w[p + "ff2.b"] = S3(f32(p + "ff.net.2.weight")), f32(p + "ff.net.2.bias")
        w["norm_out.g"], w["norm_out.b"] = f32("norm_out.weight"), f32("norm_out.bias")
        self._opad = _pad64(c.out_dim)
        w["proj_out.w3"] = S3(f32("proj_out.weight"), npad=self._opad)
        b = torch.zeros(self._opad, dtype=torch.float32, device=dev)
        b[: c.out_dim].copy_(f32("proj_out.bias"))
        w["proj_out.b"] = b
        return w

    @ops.on_device
    def init_random_(self, seed: int = 1236) -> None:
        """Synthetic weights for benchmarks (no checkpoints offline): torch default Linear/LayerNorm inits, residual-branch
        output projections scaled by 1/sqrt(num_layers + 1), generated on the GPU."""
        c = self.config
        D = c.width
        sd = SyntheticWeights(seed, self._device)
        sd.linear("post_quant", D, c.latent_channels)
        sd.linear("proj_query", D, c.query_dim)
        sd.linear("proj_out", c.out_dim, D)
        sd.layernorm("norm_out", D)
        for i in range(c.num_layers + 1):
            query = i == c.num_layers
            sd.dit_block(f"blocks.{i}.", D, 4 * D, 1.0 / math.sqrt(c.num_layers + 1), ("x_attn" if query else "s_attn",),
                         norm_cross=query)
        self.load_state_dict(sd)

    # ------------------------------------------------------------------ reference helper (temporal_autoencoder.py:118-141)
    def apply_displacement(self, vertex: torch.Tensor, displacement: torch.Tensor, scale: float = 1.0) -> torch.Tensor:
        if self.prediction_mode == "direct":
            return torch.clamp(displacement, min=-1.0 * scale, max=1.0 * scale)
        if self.prediction_mode == "residual":
            return torch.clamp(vertex[:, None] + displacement, min=-1.0 * scale, max=1.0 * scale)
        raise ValueError(f"Invalid prediction_mode: {self.prediction_mode}")

    # ------------------------------------------------------------------ forward
    def __call__(self, *args, **kwargs):
        return self.forward(*args, **kwargs)

    @ops.on_device
    @torch.no_grad()
    def forward(self, latent: torch.Tensor, framestep: torch.Tensor, source_alpha: torch.Tensor,
                target_alphas: torch.Tensor, query: torch.Tensor,
                step_callback: Optional[Callable[[int, int], None]] = None) -> torch.Tensor:
        """temporal_autoencoder.py:163-269.  latent (B,T,N,C), framestep (B,T) [any device], source_alpha (B,),
        target_alphas (B,T_out), query (B,V,3|6) -> displacement field (B,T_out,V,out_dim) fp32 in [-1,1]."""
        self._check_loaded()
        assert target_alphas.ndim == 2 and source_alpha.ndim == 1
        c, w, dev = self.config, self._w, self._device
        B, T, N, C = latent.shape
        T_out = target_alphas.shape[1]
        V = query.shape[1]
        D, H, dh = c.width, c.num_attention_heads, c.head_dim
        L = N + 1
        R = T * L                      # tokens of the trunk sequence == keys of the query cross-attention
        Rp = _pad64(R)
        scale = 1.0 / math.sqrt(dh)
        src_a = source_alpha.detach().to("cpu", torch.float32).tolist()
        tgt_a = target_alphas.detach().to("cpu", torch.float32).tolist()
        fs = framestep.detach().to("cpu", torch.float32)
        pos = fs - fs.min(dim=1, keepdim=True).values           # embeddings.py:135-153 (center=True, scale=False)
        inv = 1.0 / (10000.0 ** (torch.arange(0, dh, 2, dtype=torch.float32) / dh))
        out = torch.empty(B, T_out, V, c.out_dim, dtype=torch.float32, device=dev)

        bf, f32 = torch.bfloat16, torch.float32
        E = lambda *s, dtype=bf: torch.empty(*s, dtype=dtype, device=dev)
        lat_proj, h = E(R, D, dtype=f32), E(R, D, dtype=f32)
        xn, qkv, att, ff = E(R, D), E(R, 3 * D), E(R, D), E(R, 4 * D)
        # query-path buffers (fp32 + split operands)
        Vc = min(V, self.QUERY_CHUNK)
        qp, x1, t32 = E(V, D, dtype=f32), E(V, D, dtype=f32), E(V, D, dtype=f32)
        a3 = E(V, 3 * D)
        q3 = E(V, 3 * D)                                     # (V, H, [hi|lo|hi] x 128)
        ff32, ff3 = E(V, 4 * D, dtype=f32), E(V, 12 * D)
        ctx32 = E(R, D, dtype=f32)
        ctx3 = torch.zeros(Rp, 3 * D, dtype=bf, device=dev)  # pad rows stay zero -> K rows / V^T columns of zeros
        k32, k3 = E(Rp, D, dtype=f32), E(Rp, 3 * D)
        vt32, vt3 = E(D, Rp, dtype=f32), E(D, 3 * Rp)
        s32, p3 = E(Vc, Rp, dtype=f32), E(Vc, 3 * Rp)
        o32 = E(V, D, dtype=f32)
        logits = E(V, self._opad, dtype=f32)
        pq = f"blocks.{c.num_layers}."

        for b in range(B):
            ph = torch.outer(pos[b], inv)
            rope_cos, rope_sin = ph.cos().to(dev).contiguous(), ph.sin().to(dev).contiguous()
            rope = dict(rope_cols=2 * D, cos=rope_cos, sin=rope_sin, rows_per_pos=L)
            # post_quant (temporal_autoencoder.py:208): rows (t, n) -> trunk rows (t, n) of the [N latents | alpha] frames
            lat_bf = ops.cast_bf16(latent[b].detach().to(device=dev, dtype=f32).contiguous().view(T * N, C))
            ops.gemm(lat_bf, w["post_quant.w"], lat_proj, bias=w["post_quant.b"], row_map=(N, L, 0))
            # target-independent half of the query path: embed -> proj_query -> LN -> to_q (fp32-grade)
            pts = query[b].detach().to(device=dev, dtype=f32).contiguous()
            qe = ops.point_embedding(pts, c.embed_frequency, c.embed_include_pi, self._qpad)
            qe3 = ops.split3(qe, E(V, 3 * self._qpad))
            ops.gemm(qe3, w["proj_query.w3"], qp, bias=w["proj_query.b"], tag="s2_q")
            ops.layernorm(qp, w[pq + "norm_x_attn.g"], w[pq + "norm_x_attn.b"], 1e-5, out=t32)
            ops.split3(t32, a3)
            ops.gemm(a3, w[pq + "x.q3"], x1, tag="s2_q")                      # x1 used as scratch for q (fp32)
            ops.split3(x1, q3, seg=dh)
            for i in range(T_out):
                if step_callback is not None:
                    step_callback(i + 1, T_out)
                # ---- trunk input: projected latents + this target's alpha token per frame (:233-237,256)
                h.copy_(lat_proj)
                ops.alpha_rows(src_a[b], tgt_a[b][i], D // 2, h.view(T, L, D)[:, N, :])
                for l in range(c.num_layers):
                    blocks.attention_half(w, f"blocks.{l}.", h, xn, qkv, att, (1, R), H, norm=rope, tag="s2_gemm",
                                          attn_tag="s2_attn")
                    blocks.output_half(w, f"blocks.{l}.", "s", h, att, xn, ff, tag="s2_gemm")
                # ---- K, V^T of the query cross-attention from the trunk output (norm_cross = layer_norm, :101)
                ops.layernorm(h, w[pq + "norm_cross.g"], w[pq + "norm_cross.b"], 1e-5, out=ctx32)
                ops.split3(ctx32, ctx3)                                        # writes rows [0, R); pad rows remain 0
                ops.gemm(ctx3, w[pq + "x.k3"], k32, tag="s2_q")                # K   (Rp, D)  fp32
                ops.split3(k32, k3, seg=dh, weight=True)                       # (Rp, H, [hi|hi|lo] x 128)
                ops.gemm(w[pq + "x.v3"], ctx3, vt32, tag="s2_q")               # V^T (D, Rp)  fp32
                ops.split3(vt32, vt3, weight=True)                             # (D, [hi|hi|lo] x Rp)
                # ---- attention, unfused per head: S = q k^T -> softmax -> P v, all split-bf16 with fp32 accumulation
                for v0 in range(0, V, Vc):
                    nv = min(Vc, V - v0)
                    for hd in range(H):
                        ops.gemm(q3[v0:v0 + nv, hd * 3 * dh:(hd + 1) * 3 * dh], k3[:, hd * 3 * dh:(hd + 1) * 3 * dh],
                                 s32[:nv], tag="s2_q")
                        ops.softmax_split3(s32[:nv], R, scale, p3[:nv])
                        ops.gemm(p3[:nv], vt3[hd * dh:(hd + 1) * dh], o32[v0:v0 + nv, hd * dh:(hd + 1) * dh], tag="s2_q")
                # ---- to_out + residual, FF, output head (block.py:146-152; temporal_autoencoder.py:155-160)
                ops.split3(o32, a3)
                ops.gemm(a3, w[pq + "x.o3"], x1, bias=w[pq + "x.o.b"], residual=qp, tag="s2_q")
                ops.layernorm(x1, w[pq + "norm_ff.g"], w[pq + "norm_ff.b"], 1e-5, out=t32)
                ops.split3(t32, a3)
                ops.gemm(a3, w[pq + "ff1.w3"], ff32, bias=w[pq + "ff1.b"], act=1, tag="s2_q")
                ops.split3(ff32, ff3)
                ops.gemm(ff3, w[pq + "ff2.w3"], x1, bias=w[pq + "ff2.b"], residual=x1, tag="s2_q")
                ops.layernorm(x1, w["norm_out.g"], w["norm_out.b"], 1e-5, out=t32)
                ops.split3(t32, a3)
                ops.gemm(a3, w["proj_out.w3"], logits, bias=w["proj_out.b"], tag="s2_q")
                ops.displacement_out(logits, c.out_dim, out[b, i])
        return out
