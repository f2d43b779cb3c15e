"""B200Denoiser — sm_90a (H100) implementation of ActionMesh's temporal 3D DiT denoiser behind the reference's duck type.

Mirrors `ActionMeshDenoiser` (reference actionmesh/model/temporal_denoiser.py:23-249): same constructor fields, same
state-dict keys (SURVEY A.1), same `forward(hidden_states, context, framestep, diffusion_time, mask, freqs_rot)` ->
`(out (B,T,N,C), freqs_rot)` contract that `SchedulerFlow._diffusion_forward` calls (scheduler.py:151-158), plus
`.device / .eval() / .to() / from_pretrained()` used by the pipeline (pipeline.py:171-184).

All arithmetic runs in hand-written CUDA kernels through the C ABI (actionmesh_b200.ops); torch only owns the device
buffers.  Layout in HBM (default config, B=2 CFG branches, T=16, L=N+1=2049, D=2048, M=B*T*L=65 568 token rows):
    h      (M, D)   bf16  residual stream, rows ordered (b, t, l); row l=0 of every frame is the time token
    xn     (M, D)   bf16  LayerNorm output feeding the next GEMM
    qkv    (M, 3D)  bf16  fused [Q|K|V] with standard head order (weights are re-packed once, SURVEY A.2)
    att    (M, D)   bf16  attention output in (b, s, h, d) order == row-major (M, D)
    ff     (M, F)   bf16  GELU(MLP1)
    skips  10 x (M, D) bf16 U-ViT long-skip stack
The per-window `WindowState` returned in place of `freqs_rot` carries the RoPE tables AND the step-invariant context
K/V of all 21 cross-attention layers (SURVEY A.5), exactly the role the reference gives `freqs_rot` (an opaque cache the
scheduler threads through its loop, scheduler.py:204,224-232).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Optional

import torch

from . import ops
from ._lib import AmbError
from .blocks import SyntheticWeights, V, W, pack_block
from .blocks import repack_cross_kv, repack_self_qkv  # noqa: F401  (also importable from here, where callers import them)
from .module import B200Module


@dataclass
class DenoiserConfig:
    """Same fields/defaults as ActionMeshDenoiser's dataclass (temporal_denoiser.py:29-49)."""
    num_tokens_nominal: int = 2048
    temporal_context_size: int = 16
    in_channels: int = 64
    num_layers: int = 21
    num_attention_heads: int = 16
    width: int = 2048
    mlp_ratio: float = 4.0
    cross_attention_dim: int = 1024
    inflated_layers: tuple = field(default_factory=lambda: tuple(range(21)))

    @property
    def head_dim(self) -> int:
        return self.width // self.num_attention_heads

    @property
    def ff_dim(self) -> int:
        return int(self.width * self.mlp_ratio)


class WindowState:
    """Opaque per-window cache returned in the `freqs_rot` slot: RoPE tables + context K/V of every layer."""

    def __init__(self):
        self.rope_cos: Optional[torch.Tensor] = None   # (B*T, d_h/2) fp32
        self.rope_sin: Optional[torch.Tensor] = None
        self.ctx_kv: list[Optional[torch.Tensor]] = []  # per layer (B*T*S_ctx, 2*D) bf16, [K normed | V]
        self.ctx_zero: list[bool] = []                  # per batch element: context identically zero (A.5)
        self.shape = None
        self.source = None                              # identity of the (context, framestep) this state was built from


class B200Denoiser(B200Module):
    """Drop-in for ActionMeshDenoiser on the Stage-I hot path (inference only)."""

    config_class = DenoiserConfig

    def __init__(self, config: Optional[DenoiserConfig] = None, residual_fp32: bool = True, **kwargs):
        """`residual_fp32`: keep the residual stream (and the LayerNorm inputs) in fp32 instead of the bf16 the
        reference's autocast recipe gives it (SURVEY A.3).  GEMM / attention operands are bf16 either way; the fp32
        stream removes the 63 bf16 roundings of `h` per forward, which dominate the distance to the fp32 reference
        path (tests/test_chamfer_gpu.py measures both), for ~2 % more HBM traffic per step."""
        self.config = config if config is not None else DenoiserConfig(**kwargs)
        self.residual_fp32 = bool(residual_fp32)
        c = self.config
        if c.head_dim != 128:
            raise AmbError(f"B200Denoiser: head_dim must be 128 (width {c.width} / heads {c.num_attention_heads})")
        if c.width % 256 or c.in_channels % 64 or c.cross_attention_dim % 64:
            raise AmbError("B200Denoiser: width must be a multiple of 256, in_channels/cross_attention_dim of 64")
        super().__init__()
        self.out_channels = c.in_channels
        self._ws: dict = {}         # workspaces keyed by (B, T, N)

    def _after_to(self, moved: bool) -> None:
        if moved:
            self._ws = {}

    # ------------------------------------------------------------------ the 21 blocks as a launch program
    def _block_program(self, ws: dict, st: WindowState, b0: int, nb: int, B: int, T: int, N: int, shard):
        """Generator launching the 21 blocks (block.py:110-154) for CFG branches [b0, b0+nb) of a window: rows
        [b0*T*L, (b0+nb)*T*L) of every workspace buffer; T = the frames this rank holds.

        Single GPU: ONE program over all branches (shard None), it never yields.  Frame-sharded window: one program per
        branch; each yields right after launching its branch's K/V all-gather (and the Q projection, which does not depend
        on it) and the caller round-robins the programs, so the gather of branch b, layer l is in flight while the other
        branch runs its attention + MLP.  The last block's output is left in ws['h'] for the output head.

        U-ViT long skips (temporal_denoiser.py:222-232) never copy a residual stream: with the bf16 stream a pushing block
        writes its output straight into a skip buffer, which then serves as the read-only residual input of the next
        block; with the fp32 stream (`residual_fp32`) the stream stays in ws['h'] and the skip buffer receives the bf16
        GEMM-operand copy that `linear_skip(cat[skip, h])` needs anyway."""
        c = self.config
        w = self._w
        D, H, dh = c.width, c.num_attention_heads, c.head_dim
        L = N + 1
        TL = T * L
        f32 = self.residual_fp32
        rows = slice(b0 * TL, (b0 + nb) * TL)
        scale = 1.0 / math.sqrt(dh)
        h, xn, tmp = ws["h"][rows], ws["xn"][rows], ws["tmp"][rows]
        hb = ws["hb"][rows] if f32 else None
        qkv, att, ff = ws["qkv"][rows], ws["att"][rows], ws["ff"][rows]
        rope_cos, rope_sin = st.rope_cos[b0 * T:(b0 + nb) * T], st.rope_sin[b0 * T:(b0 + nb) * T]
        skips = [sk[rows] for sk in ws["skips"]]
        sharded = shard is not None and shard.world > 1
        if sharded:
            assert nb == 1
            kv_all = ws["kv_all"][b0]                                           # kv_all[b]: (world, TL, 2D)
        S = st.ctx_kv[0].shape[0] // (B * T)
        sp = 0
        half = c.num_layers // 2
        h_in = h  # where the current residual stream lives
        for i in range(c.num_layers):
            p = f"blocks.{i}."
            if i > half:  # block.py:131-133: LN(W_skip [skip | h] + b) without materialising the concat
                sp -= 1
                # fp32 stream: its bf16 GEMM-operand copy was written by the previous block's last GEMM (second output)
                ops.gemm(skips[sp], w[p + "skip.w"], tmp, a2=hb if f32 else h_in, bias=w[p + "skip.b"])
                ops.layernorm(tmp, w[p + "norm_skip.g"], w[p + "norm_skip.b"], 1e-5, out=h)
                h_in = h
            # ---- self-attention (block.py:137-142, attention_processor.py:49-166)
            ops.layernorm(h_in, w[p + "norm_s_attn.g"], w[p + "norm_s_attn.b"], 1e-5, out=xn)
            inflated = i in c.inflated_layers
            if sharded and inflated:
                # this exchange's send buffer (a shard exchanging over peer memory double-buffers it, window_shard.py)
                kv_local = shard.kv_local_view(ws["kv_local"], rows, b0) if hasattr(shard, "kv_local_view") else ws["kv_local"][rows]
                ops.gemm(xn, w[p + "s.qkv"][D:], kv_local,
                         norm=dict(cols=D, seg=D, w0=w[p + "s.nk"], eps=1e-6, rope_cols=D, cos=rope_cos, sin=rope_sin,
                                   rows_per_pos=L))
                work = shard.all_gather_kv(kv_all.view(-1, 2 * D), kv_local, b0)
                ops.gemm(xn, w[p + "s.qkv"][:D], qkv[:, 0:D],
                         norm=dict(cols=D, seg=D, w0=w[p + "s.nq"], eps=1e-6, rope_cols=D, cos=rope_cos, sin=rope_sin,
                                   rows_per_pos=L))
                yield
                work.wait()
                k5 = kv_all[None, :, :, 0:D].unflatten(-1, (H, dh))
                v5 = kv_all[None, :, :, D:2 * D].unflatten(-1, (H, dh))
                ops.flash_attn(qkv[:, 0:D].unflatten(-1, (H, dh))[None], k5, v5, att.view(1, TL, H, dh), scale,
                               kv_chunks=shard.world, tag="attn_self")
            else:
                ops.gemm(xn, w[p + "s.qkv"], qkv,
                         norm=dict(cols=2 * D, seg=D, w0=w[p + "s.nq"], w1=w[p + "s.nk"], eps=1e-6, rope_cols=2 * D,
                                   cos=rope_cos, sin=rope_sin, rows_per_pos=L))
                view = (nb, TL, H, dh) if inflated else (nb * T, L, H, dh)
                q4, k4, v4 = (qkv[:, j * D:(j + 1) * D].unflatten(0, view[:2]).unflatten(-1, (H, dh)) for j in range(3))
                ops.flash_attn(q4, k4, v4, att.view(*view), scale, tag="attn_self")
            ops.gemm(att, w[p + "s.o.w"], h, bias=w[p + "s.o.b"], residual=h_in)
            h_in = h
            # ---- cross-attention (block.py:146-149); zero-context batch elements reduce to + to_out.0.bias (A.5)
            for b in range(b0, b0 + nb):
                r = slice((b - b0) * TL, (b - b0 + 1) * TL)
                if st.ctx_zero[b]:
                    ops.add_bias_rows(h[r], w[p + "x.o.b"])
                    continue
                ops.layernorm(h[r], w[p + "norm_x_attn.g"], w[p + "norm_x_attn.b"], 1e-5, out=xn[r])
                qb = qkv[r, 0:D]
                ops.gemm(xn[r], w[p + "x.q"], qb, norm=dict(cols=D, seg=D, w0=w[p + "x.nq"], eps=1e-6))
                kvb = st.ctx_kv[i][b * T * S:(b + 1) * T * S]
                ops.flash_attn(qb.view(T, L, H, dh), kvb[:, 0:D].view(T, S, H, dh), kvb[:, D:2 * D].view(T, S, H, dh),
                               att[r].view(T, L, H, dh), scale, tag="attn_cross")
                ops.gemm(att[r], w[p + "x.o.w"], h[r], bias=w[p + "x.o.b"], residual=h[r])
            # ---- feed-forward (block.py:152)
            ops.layernorm(h, w[p + "norm_ff.g"], w[p + "norm_ff.b"], 1e-5, out=xn)
            ops.gemm(xn, w[p + "ff1.w"], ff, bias=w[p + "ff1.b"], act=1)
            if i < half and not f32:  # temporal_denoiser.py:231-232: push == write the block output into the skip buffer
                ops.gemm(ff, w[p + "ff2.w"], skips[sp], bias=w[p + "ff2.b"], residual=h)
                h_in = skips[sp]
                sp += 1
            else:
                # fp32 stream: the stream stays in h; the second (bf16) output is the operand `linear_skip(cat[skip, h])`
                # needs — the skip itself for a pushing block, the h half for the block before a popping one
                copy = skips[sp] if i < half else (hb if (f32 and half <= i < c.num_layers - 1) else None)
                ops.gemm(ff, w[p + "ff2.w"], h, bias=w[p + "ff2.b"], residual=h, out2=copy)
                if i < half:
                    sp += 1
        assert h_in is h  # the last block is never a pushing block: its output lives in ws['h'] for the output head

    # ------------------------------------------------------------------ weights
    def _pack_state_dict(self, sd: dict, dev: torch.device) -> dict:
        """Pack the reference's state dict (keys of SURVEY A.1) into kernel-ready tensors: GEMM weights bf16 (QKV / KV
        fused and head-permuted), biases / norm weights fp32."""
        w = {}
        w["proj_in.w"], w["proj_in.b"] = W(sd["proj_in.weight"], dev), V(sd["proj_in.bias"], dev)
        w["time1.w"], w["time1.b"] = W(sd["time_proj.linear_1.weight"], dev), V(sd["time_proj.linear_1.bias"], dev)
        w["time2.w"], w["time2.b"] = W(sd["time_proj.linear_2.weight"], dev), V(sd["time_proj.linear_2.bias"], dev)
        w["norm_out.g"], w["norm_out.b"] = V(sd["norm_out.weight"], dev), V(sd["norm_out.bias"], dev)
        w["proj_out.w"], w["proj_out.b"] = W(sd["proj_out.weight"], dev), V(sd["proj_out.bias"], dev)
        for i in range(self.config.num_layers):
            pack_block(w, sd, f"blocks.{i}.", f"blocks.{i}.", self.config.num_attention_heads, dev)
        return w

    def init_random_(self, seed: int = 1234, residual_scale: Optional[float] = None) -> None:
        """Synthetic weights for benchmarks (no checkpoints offline): torch default Linear/LayerNorm inits, residual
        branch output projections scaled by 1/sqrt(num_layers) so activations stay O(1) (SURVEY 8(d)).  Generated
        directly on the GPU (no 5.8 GB host copy)."""
        c = self.config
        rs = residual_scale if residual_scale is not None else 1.0 / math.sqrt(c.num_layers)
        sd = SyntheticWeights(seed, self._device)
        sd.linear("proj_in", c.width, c.in_channels)
        sd.linear("time_proj.linear_1", c.width * 4, c.width)
        sd.linear("time_proj.linear_2", c.width, c.width * 4)
        sd.layernorm("norm_out", c.width)
        sd.linear("proj_out", c.in_channels, c.width)
        for i in range(c.num_layers):
            sd.dit_block(f"blocks.{i}.", c.width, c.ff_dim, rs, ("s_attn", "x_attn"), cross_dim=c.cross_attention_dim,
                         qk_norm=c.head_dim, skip=i > c.num_layers // 2)
        self.load_state_dict(sd)
        del sd
        torch.cuda.empty_cache()

    # ------------------------------------------------------------------ workspaces
    def _workspace(self, B: int, T: int, N: int, world: int = 1, slot: int = 0, shard=None) -> dict:
        """Activation buffers of one window shape.  `slot` > 0 gives additional independent sets of the same shape (the
        single-GPU emulation of several ranks in tests/test_window_shard_gpu.py); one shape stays resident."""
        symmetric = shard is not None and hasattr(shard, "empty_kv_local")   # the exchange decides where kv_local lives
        key = (B, T, N, world, slot, id(shard) if symmetric else 0)
        ws = self._ws.get(key)
        if ws is not None:
            return ws
        c = self.config
        dev = self._device
        L = N + 1
        M = B * T * L
        bf = torch.bfloat16
        hd = torch.float32 if self.residual_fp32 else bf
        n_skips = c.num_layers // 2
        ws = {
            "x_in": torch.empty(B * T * N, c.in_channels, dtype=bf, device=dev),
            "t_emb": torch.empty(B * T, c.width, dtype=bf, device=dev),
            "t_hid": torch.empty(B * T, c.width * 4, dtype=bf, device=dev),
            "h": torch.empty(M, c.width, dtype=hd, device=dev),
            "xn": torch.empty(M, c.width, dtype=bf, device=dev),
            "tmp": torch.empty(M, c.width, dtype=hd, device=dev),
            "hb": torch.empty(M, c.width, dtype=bf, device=dev) if self.residual_fp32 else None,
            "qkv": torch.empty(M, 3 * c.width, dtype=bf, device=dev),
            "att": torch.empty(M, c.width, dtype=bf, device=dev),
            "ff": torch.empty(M, c.ff_dim, dtype=bf, device=dev),
            "skips": [torch.empty(M, c.width, dtype=bf, device=dev) for _ in range(n_skips)],
            "pred": torch.empty(M, c.in_channels, dtype=bf, device=dev),
        }
        if world > 1:  # frame-sharded window: local [K|V] rows and the all-gathered buffer (one chunk per rank)
            if symmetric:
                ws["kv_local"] = shard.empty_kv_local(M, 2 * c.width, dev)     # symmetric memory mapped into every peer
            else:
                ws["kv_local"] = torch.empty(M, 2 * c.width, dtype=bf, device=dev)
            ws["kv_all"] = torch.empty(B, world, T * L, 2 * c.width, dtype=bf, device=dev)
        self._ws = {k: v for k, v in self._ws.items() if k[:4] == key[:4]}  # keep one shape resident
        self._ws[key] = ws
        return ws

    # ------------------------------------------------------------------ per-window cache
    def precompute_window(self, context: torch.Tensor, framestep: torch.Tensor, N: int,
                          frame_slice: Optional[slice] = None) -> WindowState:
        """Step-invariant work of one AR window: RoPE tables (temporal_denoiser.py:114-149) and, for every layer,
        K = norm_k(to_k(ctx)), V = to_v(ctx) of the cross-attention (attention_processor.py:101-124).  Batch elements
        whose context is identically zero (the CFG "no image" branch, guidance.py:73) are flagged so their
        cross-attention collapses to `to_out.0.bias` (SURVEY A.5); that check is the only host sync, once per window."""
        c = self.config
        dev = self._device
        # RoPE: theta_j = 10000^(-2j/d_h); phase = (framestep - min) * theta_j   (rotary_embedding.py:42-58).  With a
        # frame-sharded window the minimum is taken over the WHOLE window, then this rank's frames are selected.
        fs = framestep.detach().to("cpu", torch.float32)
        pos = fs - fs.min(dim=1, keepdim=True).values
        if frame_slice is not None:
            pos = pos[:, frame_slice]
            context = context[:, frame_slice]
        B, T, S, Dc = context.shape
        st = WindowState()
        st.shape = (B, T, N)
        pos = pos.reshape(B * T)
        inv = 1.0 / (10000.0 ** (torch.arange(0, c.head_dim, 2, dtype=torch.float32) / c.head_dim))
        ph = torch.outer(pos, inv)
        st.rope_cos = ph.cos().to(dev).contiguous()
        st.rope_sin = ph.sin().to(dev).contiguous()
        ctx = context.detach().to(device=dev, dtype=torch.float32).contiguous()
        st.ctx_zero = [bool(z) for z in (ctx.reshape(B, -1).abs().amax(dim=1) == 0).tolist()]
        ctx_bf = ops.cast_bf16(ctx.view(B * T * S, Dc))
        for i in range(c.num_layers):
            p = f"blocks.{i}."
            kv = torch.empty(B * T * S, 2 * c.width, dtype=torch.bfloat16, device=dev)
            ops.gemm(ctx_bf, self._w[p + "x.kv"], kv,
                     norm=dict(cols=c.width, seg=c.width, w0=self._w[p + "x.nk"], eps=1e-6))
            st.ctx_kv.append(kv)
        return st

    # ------------------------------------------------------------------ forward
    @ops.on_device
    @torch.no_grad()
    def forward(self, hidden_states: torch.Tensor, context: torch.Tensor, framestep: torch.Tensor,
                diffusion_time: torch.Tensor, mask: Optional[torch.Tensor] = None, freqs_rot=None):
        """ActionMeshDenoiser.forward (temporal_denoiser.py:151-249).  Returns (prediction (B,T,N,C) bf16, state).

        `freqs_rot` is the WindowState from a previous call of the same window (or None).  The prediction is a VIEW of a
        workspace buffer that the next forward() overwrites (the scheduler consumes it immediately); clone it to keep it."""
        self._check_loaded()
        B, T, N, C = hidden_states.shape
        # The state caches the image conditioning as well as the RoPE tables, so (unlike the reference's freqs_rot) it is
        # only reused for the context / framestep it was built from.
        source = (context.data_ptr(), context._version, tuple(context.shape), tuple(framestep.reshape(-1).tolist()))
        st = freqs_rot if isinstance(freqs_rot, WindowState) else None
        if st is None or st.shape != (B, T, N) or st.source != source:
            st = self.precompute_window(context, framestep, N)
            st.source = source
        x32 = hidden_states.detach().to(device=self._device, dtype=torch.float32).contiguous()
        t32 = diffusion_time.detach().to(device=self._device, dtype=torch.float32).contiguous()
        m32 = None
        if mask is not None:
            m32 = mask.detach().to(device=self._device, dtype=torch.float32).reshape(B * T).contiguous()
        ws = self._workspace(B, T, N)
        ops.cast_bf16(x32.view(B * T * N, C), out=ws["x_in"])
        pred = self._forward_packed(ws, st, B, T, N, t32, m32, n_input_branches=B)
        return pred.view(B, T, N + 1, C)[:, :, 1:, :], st

    __call__ = forward

    def _forward_packed(self, ws: dict, st: WindowState, B: int, T: int, N: int, t32: torch.Tensor,
                        m32: Optional[torch.Tensor], n_input_branches: int, shard=None) -> torch.Tensor:
        """Runs the 21-block DiT on ws['x_in'] (bf16 latents of `n_input_branches` batch elements; when fewer than B,
        the same latents feed every CFG branch) and leaves the prediction in ws['pred'] (M, C) bf16."""
        c = self.config
        w = self._w
        D, H, dh = c.width, c.num_attention_heads, c.head_dim
        L = N + 1
        M = B * T * L
        h, xn, tmp, qkv, att, ff = ws["h"], ws["xn"], ws["tmp"], ws["qkv"], ws["att"], ws["ff"]
        scale = 1.0 / math.sqrt(dh)

        # proj_in (temporal_denoiser.py:205-206): rows (bt, n) -> h rows (bt, 1 + n).  When the CFG branches share
        # their latents (guidance.py:56 `cat([latent] * K)`) the same bf16 rows feed every branch's copy.
        nb = n_input_branches
        x_in = ws["x_in"][: nb * T * N]
        for r in range(B // nb):
            ops.gemm(x_in, w["proj_in.w"], h[r * nb * T * L:], bias=w["proj_in.b"], row_map=(N, L, 1))
        # time token (temporal_denoiser.py:209-217)
        ops.timestep_embedding(t32, D, out=ws["t_emb"], mask=m32, rows=B * T)
        ops.gemm(ws["t_emb"], w["time1.w"], ws["t_hid"], bias=w["time1.b"], act=1)
        ops.gemm(ws["t_hid"], w["time2.w"], h, bias=w["time2.b"], row_map=(1, L, 0))

        # The 21 blocks: one launch program over all CFG branches on a single GPU; for a frame-sharded window the branches
        # are independent through the whole network, so they run as staggered programs on the one compute stream — while
        # branch b's K/V all-gather is in flight the other branch runs its attention / MLP (see _block_program).
        if shard is not None and shard.world > 1:
            progs = [self._block_program(ws, st, b, 1, B, T, N, shard) for b in range(B)]
        else:
            progs = [self._block_program(ws, st, 0, B, B, T, N, None)]
        live = list(progs)
        while live:
            for g in list(live):
                try:
                    next(g)
                except StopIteration:
                    live.remove(g)
        # output head (temporal_denoiser.py:239-242); the time-token rows are computed and ignored by the consumers
        ops.layernorm(h, w["norm_out.g"], w["norm_out.b"], 1e-5, out=xn)
        ops.gemm(xn, w["proj_out.w"], ws["pred"], bias=w["proj_out.b"])
        return ws["pred"]
