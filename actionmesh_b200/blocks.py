"""The pre-LN DiT block the host-side models share: weight packing, synthetic weights and its launch sequence.

Packed names, under a block prefix p (the denoiser's scheme; every model packs its blocks this way):
    norm_s_attn / norm_x_attn / norm_ff / norm_skip / norm_cross .g .b     LayerNorm weight / bias, fp32
    s.qkv                  self-attention [Q | K | V], head split folded in (repack_self_qkv), bf16
    x.q, x.kv              cross-attention Q and [K | V] (repack_cross_kv), bf16
    s.nq s.nk x.nq x.nk    per-head q / k RMSNorm weights, fp32
    s.o / x.o .w .b        attention output projection
    ff1 / ff2 .w .b        feed-forward; skip.w, skip.b the U-ViT long-skip linear

A block runs as two launch sequences over an fp32 residual stream x with bf16 operands: `attention_half` (LayerNorm ->
fused QKV GEMM -> flash attention) and `output_half` (o-proj + residual -> LayerNorm -> FF1 GELU -> FF2 + residual).  The
denoiser's blocks (skips, cross-attention, sharded K/V) keep their own launch program in denoiser.py.
"""
from __future__ import annotations

import math

import torch

from . import ops

# TripoSG DiTBlock keys (norm1/attn1/norm2/attn2/norm3/ff/skip_linear/skip_norm, triposg_transformer.py:190-262) -> the
# ActionMeshDenoiser keys (block.py:64-108)
TRIPOSG_BLOCK_KEYS = (("norm1.", "norm_s_attn."), ("attn1.", "s_attn."), ("norm2.", "norm_x_attn."), ("attn2.", "x_attn."),
                      ("norm3.", "norm_ff."), ("skip_linear.", "linear_skip."), ("skip_norm.", "norm_skip."))


def remap_block_keys(sd: dict, pairs, prefix: str = "blocks.") -> dict:
    """Keys `{prefix}{i}.{a}...` -> `{prefix}{i}.{b}...` for the first pair (a, b) whose `a` starts the block-level key;
    the other keys pass through."""
    out = {}
    for k, v in sd.items():
        if k.startswith(prefix):
            idx, rest = k[len(prefix):].split(".", 1)
            for a, b in pairs:
                if rest.startswith(a):
                    rest = b + rest[len(a):]
                    break
            k = f"{prefix}{idx}.{rest}"
        out[k] = v
    return out


def remap_triposg_state_dict(sd: dict, prefix: str = "blocks.") -> dict:
    """TripoSG DiTBlock keys under `prefix` -> the ActionMesh keys `pack_block` reads."""
    return remap_block_keys(sd, TRIPOSG_BLOCK_KEYS, prefix)


def repack_self_qkv(wq: torch.Tensor, wk: torch.Tensor, wv: torch.Tensor, heads: int) -> torch.Tensor:
    """Head-interleaved split of attention_processor.py:106-110 folded into the weights (SURVEY A.2).

    The reference takes head h's q/k/v from columns [3dh, 3d(h+1)) of cat(q,k,v).  Selecting the matching ROWS of
    cat(Wq,Wk,Wv) once gives a standard fused QKV GEMM whose output is [Q(h,d) | K(h,d) | V(h,d)]."""
    wcat = torch.cat([wq, wk, wv], dim=0)  # (3*inner, in)
    inner = wq.shape[0]
    dh = inner // heads
    wcat = wcat.view(heads, 3, dh, -1)
    return torch.cat([wcat[:, 0].reshape(inner, -1), wcat[:, 1].reshape(inner, -1), wcat[:, 2].reshape(inner, -1)], 0)


def repack_cross_kv(wk: torch.Tensor, wv: torch.Tensor, heads: int) -> torch.Tensor:
    """Same for the cross-attention [k|v] split (attention_processor.py:111-115); q keeps the plain head view (:117)."""
    wcat = torch.cat([wk, wv], dim=0)
    inner = wk.shape[0]
    dh = inner // heads
    wcat = wcat.view(heads, 2, dh, -1)
    return torch.cat([wcat[:, 0].reshape(inner, -1), wcat[:, 1].reshape(inner, -1)], 0)


def V(t: torch.Tensor, dev) -> torch.Tensor:
    """fp32 copy on `dev`: vectors, and the fp32 source of a packed matrix."""
    return t.detach().to(device=dev, dtype=torch.float32).contiguous()


def W(t: torch.Tensor, dev) -> torch.Tensor:
    """bf16 GEMM operand, rounded once from fp32."""
    return V(t, dev).to(torch.bfloat16).contiguous()


def pack_block(w: dict, sd: dict, src: str, dst: str, heads: int, dev) -> None:
    """Pack the block `src` of a state dict with ActionMesh's key names into `w` under prefix `dst`.  Each part (long
    skip, self- and cross-attention, their q/k norms, norm_cross) is packed when the block has it."""
    for n in ("norm_skip", "norm_s_attn", "norm_x_attn", "norm_ff"):
        if src + n + ".weight" in sd:
            w[dst + n + ".g"], w[dst + n + ".b"] = V(sd[src + n + ".weight"], dev), V(sd[src + n + ".bias"], dev)
    if src + "linear_skip.weight" in sd:
        w[dst + "skip.w"], w[dst + "skip.b"] = W(sd[src + "linear_skip.weight"], dev), V(sd[src + "linear_skip.bias"], dev)
    for attn, q in (("s_attn.", "s."), ("x_attn.", "x.")):
        a, q = src + attn, dst + q
        if a + "to_q.weight" not in sd:
            continue
        wq, wk, wv = (V(sd[a + f"to_{n}.weight"], dev) for n in "qkv")
        if attn == "s_attn.":
            w[q + "qkv"] = repack_self_qkv(wq, wk, wv, heads).to(torch.bfloat16).contiguous()
        else:
            w[q + "q"] = wq.to(torch.bfloat16).contiguous()
            w[q + "kv"] = repack_cross_kv(wk, wv, heads).to(torch.bfloat16).contiguous()
        if a + "norm_q.weight" in sd:
            w[q + "nq"], w[q + "nk"] = V(sd[a + "norm_q.weight"], dev), V(sd[a + "norm_k.weight"], dev)
        if a + "norm_cross.weight" in sd:
            w[dst + "norm_cross.g"], w[dst + "norm_cross.b"] = V(sd[a + "norm_cross.weight"], dev), V(sd[a + "norm_cross.bias"], dev)
        w[q + "o.w"], w[q + "o.b"] = W(sd[a + "to_out.0.weight"], dev), V(sd[a + "to_out.0.bias"], dev)
    w[dst + "ff1.w"], w[dst + "ff1.b"] = W(sd[src + "ff.net.0.proj.weight"], dev), V(sd[src + "ff.net.0.proj.bias"], dev)
    w[dst + "ff2.w"], w[dst + "ff2.b"] = W(sd[src + "ff.net.2.weight"], dev), V(sd[src + "ff.net.2.bias"], dev)


class SyntheticWeights(dict):
    """A state dict of synthetic weights for benchmarks (no checkpoints offline): torch's default Linear init
    U(±1/sqrt(in_features)) drawn from one generator on `device` in call order, LayerNorms at (1, 0)."""

    def __init__(self, seed: int, device):
        super().__init__()
        self.device = device
        self.generator = torch.Generator(device=device).manual_seed(seed)

    def linear(self, name: str, out_f: int, in_f: int, scale: float = 1.0, bias: bool = True) -> None:
        bound = 1.0 / math.sqrt(in_f)
        g, dev = self.generator, self.device
        self[name + ".weight"] = (torch.rand(out_f, in_f, generator=g, device=dev) * 2 - 1) * bound * scale
        if bias:
            self[name + ".bias"] = (torch.rand(out_f, generator=g, device=dev) * 2 - 1) * bound * scale

    def layernorm(self, name: str, width: int) -> None:
        self[name + ".weight"], self[name + ".bias"] = torch.ones(width, device=self.device), torch.zeros(width, device=self.device)

    def dit_block(self, p: str, width: int, ff_dim: int, residual_scale: float, attn=("s_attn",), *, cross_dim: int = 0,
                  qk_norm: int = 0, norm_cross: bool = False, skip: bool = False) -> None:
        """Block `p` with ActionMesh's key names: the long skip when `skip`, then per attention in `attn` q, k, v (cross
        k / v from `cross_dim` features, default `width`), `qk_norm`-wide q / k norms, norm_cross, to_out; then the
        feed-forward.  Output projections are scaled by `residual_scale`."""
        if skip:
            self.linear(p + "linear_skip", width, 2 * width)
            self.layernorm(p + "norm_skip", width)
        for a in attn:
            self.layernorm(p + "norm_" + a, width)
            kd = cross_dim if a == "x_attn" and cross_dim else width
            self.linear(p + a + ".to_q", width, width, bias=False)
            self.linear(p + a + ".to_k", width, kd, bias=False)
            self.linear(p + a + ".to_v", width, kd, bias=False)
            if qk_norm:
                self[p + a + ".norm_q.weight"] = torch.ones(qk_norm, device=self.device)
                self[p + a + ".norm_k.weight"] = torch.ones(qk_norm, device=self.device)
            if norm_cross:
                self.layernorm(p + a + ".norm_cross", width)
            self.linear(p + a + ".to_out.0", width, width, scale=residual_scale)
        self.layernorm(p + "norm_ff", width)
        self.linear(p + "ff.net.0.proj", ff_dim, width)
        self.linear(p + "ff.net.2", width, ff_dim, scale=residual_scale)


def attention_half(w: dict, p: str, x: torch.Tensor, xn: torch.Tensor, qkv: torch.Tensor, att: torch.Tensor, view, heads: int,
                   *, eps: float = 1e-5, bias=None, norm=None, tag: str, attn_tag: str) -> None:
    """LayerNorm (norm_s_attn) of x -> fused QKV GEMM (s.qkv, with the `bias` and `norm=` epilogues as given) -> flash
    attention of the rows viewed as (batch, seq) = `view` into att."""
    D = att.shape[1]
    dh = D // heads
    ops.layernorm(x, w[p + "norm_s_attn.g"], w[p + "norm_s_attn.b"], eps, out=xn)
    ops.gemm(xn, w[p + "s.qkv"], qkv, bias=bias, norm=norm, tag=tag)
    q, k, v = (qkv[:, j * D:(j + 1) * D].unflatten(0, view).unflatten(-1, (heads, dh)) for j in range(3))
    ops.flash_attn(q, k, v, att.view(*view, heads, dh), 1.0 / math.sqrt(dh), tag=attn_tag)


def output_half(w: dict, p: str, attn: str, x: torch.Tensor, att: torch.Tensor, xn: torch.Tensor, ff: torch.Tensor, *,
                eps: float = 1e-5, layer_scale=(None, None), tag: str) -> None:
    """Output projection `attn`.o (s or x) + residual -> LayerNorm (norm_ff) -> FF1 GELU -> FF2 + residual, in place on
    x; `layer_scale` = the column scales of the two residual GEMMs (DinoV2's LayerScale)."""
    ops.gemm(att, w[p + attn + ".o.w"], x, bias=w[p + attn + ".o.b"], col_scale=layer_scale[0], residual=x, tag=tag)
    ops.layernorm(x, w[p + "norm_ff.g"], w[p + "norm_ff.b"], eps, out=xn)
    ops.gemm(xn, w[p + "ff1.w"], ff, bias=w[p + "ff1.b"], act=1, tag=tag)
    ops.gemm(ff, w[p + "ff2.w"], x, bias=w[p + "ff2.b"], col_scale=layer_scale[1], residual=x, tag=tag)
