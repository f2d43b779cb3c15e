"""B200AttentionProcessor — drop-in for the reference's diffusers attention-processor plugin (seam 1).

Same call signature as `AttentionProcessor.__call__` (actionmesh/model/utils/attention_processor.py:36-46).  It reads the
diffusers `Attention` container it is attached to (`to_q/to_k/to_v/to_out[0]/norm_q/norm_k/heads/is_cross_attention`)
and runs the whole processor body on the sm_90a kernels: fused-QKV wgmma GEMM whose epilogue does the
head-interleaved split (folded into a one-time weight permutation), RMS qk-norm and RoPE; wgmma flash attention;
to_out GEMM with bias.  Returns a NEW tensor of the input dtype and never aliases the (normed) input, as the block
relies on (`hidden_states + self.s_attn(self.norm_s_attn(hidden_states))`, block.py:137).

Packed weights are cached on the processor instance keyed by the parameter storage, so the permutation/cast happens once
per module (inference; weights frozen).
"""
from __future__ import annotations

import math
from typing import Optional

import torch

from . import ops
from ._lib import AmbError
from .blocks import repack_cross_kv, repack_self_qkv


class B200AttentionProcessor:
    def __init__(self):
        self._cache = {}

    def invalidate(self) -> None:
        """Drop every packed-weight entry (e.g. after swapping parameter tensors of the modules this processor serves)."""
        self._cache.clear()

    def _packed(self, attn):
        # one entry per module (a processor instance may be shared by all layers); the key carries the pointers AND the
        # in-place version counters of every weight that is packed, so load_state_dict / copy_ re-packs
        params = [attn.to_q.weight, attn.to_k.weight, attn.to_v.weight, attn.to_out[0].weight]
        params += [t for t in (getattr(attn.norm_q, "weight", None), getattr(attn.norm_k, "weight", None), attn.to_out[0].bias)
                   if t is not None]
        key = tuple((t.data_ptr(), t._version, t.device) for t in params)
        hit = self._cache.get(id(attn))
        if hit is not None and hit[0] == key:
            return hit[1]
        for name in ("to_q", "to_k", "to_v"):
            if getattr(attn, name).bias is not None:
                raise AmbError("B200AttentionProcessor: q/k/v bias unsupported (reference uses attention_bias=False)")
        if attn.norm_q is None or attn.norm_k is None:
            raise AmbError("B200AttentionProcessor: requires qk_norm='rms_norm' (reference default)")
        dev = attn.to_q.weight.device
        f32 = lambda t: t.detach().to(device=dev, dtype=torch.float32)
        H = attn.heads
        w = {}
        if attn.is_cross_attention:
            w["q"] = f32(attn.to_q.weight).to(torch.bfloat16).contiguous()
            w["kv"] = repack_cross_kv(f32(attn.to_k.weight), f32(attn.to_v.weight), H).to(torch.bfloat16).contiguous()
        else:
            w["qkv"] = repack_self_qkv(f32(attn.to_q.weight), f32(attn.to_k.weight), f32(attn.to_v.weight),
                                       H).to(torch.bfloat16).contiguous()
        w["nq"], w["nk"] = f32(attn.norm_q.weight).contiguous(), f32(attn.norm_k.weight).contiguous()
        w["eps"] = float(getattr(attn.norm_q, "eps", 1e-6))
        w["o.w"] = f32(attn.to_out[0].weight).to(torch.bfloat16).contiguous()
        w["o.b"] = f32(attn.to_out[0].bias).contiguous() if attn.to_out[0].bias is not None else None
        self._cache[id(attn)] = (key, w)
        return w

    @torch.no_grad()
    def __call__(self, attn, hidden_states: torch.Tensor, encoder_hidden_states: Optional[torch.Tensor] = None,
                 attention_mask: Optional[torch.Tensor] = None, temb: Optional[torch.Tensor] = None,
                 inflate_self_attention: bool = False, freqs_rot=None, n_frames: Optional[int] = None) -> torch.Tensor:
        if attention_mask is not None:
            raise AmbError("B200AttentionProcessor: attention_mask is not used on the ActionMesh path")
        if not hidden_states.is_cuda:
            raise AmbError("B200AttentionProcessor: CUDA tensors only (no CPU fallback)")
        if getattr(attn, "residual_connection", False) or getattr(attn, "rescale_output_factor", 1.0) != 1.0:
            raise AmbError("B200AttentionProcessor: residual_connection / rescale_output_factor unsupported")
        w = self._packed(attn)
        in_dtype = hidden_states.dtype
        BT, Lq, D = hidden_states.shape
        H = attn.heads
        dh = D // H
        if dh != 128:
            raise AmbError("B200AttentionProcessor: head_dim must be 128")
        dev = hidden_states.device
        x = hidden_states.reshape(BT * Lq, D)
        x = x if x.dtype == torch.bfloat16 else ops.cast_bf16(x.float().contiguous())
        M = BT * Lq
        att = torch.empty(M, D, dtype=torch.bfloat16, device=dev)
        scale = 1.0 / math.sqrt(dh)
        if not attn.is_cross_attention:
            if encoder_hidden_states is not None:
                raise AmbError("self-attention container called with encoder_hidden_states")
            norm = dict(cols=2 * D, seg=D, w0=w["nq"], w1=w["nk"], eps=w["eps"])
            if freqs_rot is not None:
                cos, sin = freqs_rot  # (BT, L, dh) with repeat_interleave(2) pairs, constant per frame
                norm.update(rope_cols=2 * D, cos=cos[:, 0, 0::2].float().contiguous(),
                            sin=sin[:, 0, 0::2].float().contiguous(), rows_per_pos=Lq)
            qkv = torch.empty(M, 3 * D, dtype=torch.bfloat16, device=dev)
            ops.gemm(x, w["qkv"], qkv, norm=norm)
            if inflate_self_attention:
                assert n_frames is not None
                view = (BT // n_frames, n_frames * Lq)
            else:
                view = (BT, Lq)
            q4 = qkv[:, 0:D].unflatten(0, view).unflatten(-1, (H, dh))
            k4 = qkv[:, D:2 * D].unflatten(0, view).unflatten(-1, (H, dh))
            v4 = qkv[:, 2 * D:].unflatten(0, view).unflatten(-1, (H, dh))
            ops.flash_attn(q4, k4, v4, att.view(*view, H, dh), scale)
        else:
            ctx = encoder_hidden_states
            S, Dc = ctx.shape[1], ctx.shape[2]
            c = ctx.reshape(BT * S, Dc)
            c = c if c.dtype == torch.bfloat16 else ops.cast_bf16(c.float().contiguous())
            q = torch.empty(M, D, dtype=torch.bfloat16, device=dev)
            kv = torch.empty(BT * S, 2 * D, dtype=torch.bfloat16, device=dev)
            ops.gemm(x, w["q"], q, norm=dict(cols=D, seg=D, w0=w["nq"], eps=w["eps"]))
            ops.gemm(c, w["kv"], kv, norm=dict(cols=D, seg=D, w0=w["nk"], eps=w["eps"]))
            ops.flash_attn(q.view(BT, Lq, H, dh), kv[:, 0:D].view(BT, S, H, dh), kv[:, D:].view(BT, S, H, dh),
                           att.view(BT, Lq, H, dh), scale)
        out = torch.empty(M, D, dtype=torch.bfloat16 if in_dtype == torch.bfloat16 else torch.float32, device=dev)
        ops.gemm(att, w["o.w"], out, bias=w["o.b"])
        return out.view(BT, Lq, D).to(in_dtype)
