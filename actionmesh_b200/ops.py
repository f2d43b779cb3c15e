"""Torch-tensor front door to the C ABI (device pointers + the current CUDA stream; torch is only plumbing here).

Every function launches hand-written sm_90a kernels from libactionmesh_b200.so; nothing here computes with torch ops.
Each wrapper hands every tensor to the ABI through `_ptr` (CUDA, dtype, current device -> device pointer) and makes its
ABI calls through `_launch`, which appends the current stream, raises AmbError on a non-zero return, adds the wrapper's
kernel count to the global `launch_count` (so bench.py can report how many of OUR kernels ran in the timed region) and,
for a tagged call, records CUDA events into `event_log`.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _lib

launch_count = 0

# Optional per-kernel CUDA-event timing (bench.py's roofline legs): when `event_log` is a list, launches whose `tag` is
# in `event_tags` append (tag, start_event, end_event, meta) recorded on the launching stream; meta = the launch's shape.
event_log = None
event_tags: set = set()

_FLOAT = (torch.bfloat16, torch.float32)


def on_device(fn):
    """Method decorator for the module-level entry points: makes `self.device` the current CUDA device for the call (the C
    ABI launches on the current device and stream)."""
    import functools

    @functools.wraps(fn)
    def wrapper(self, *args, **kwargs):
        dev = self.device
        if dev.type != "cuda":
            return fn(self, *args, **kwargs)
        with torch.cuda.device(dev):
            return fn(self, *args, **kwargs)

    return wrapper


class _Abi:
    """The library's functions as attributes, each looked up once (the library loads on first use, not on import)."""

    def __getattr__(self, name):
        fn = getattr(_lib.load_library(), name)
        setattr(self, name, fn)
        return fn


_abi = _Abi()


def _launch(fn, kernels: int, *args, tag: Optional[str] = None, meta=None) -> None:
    """fn(*args, current stream), raising AmbError on a non-zero return; adds `kernels` to launch_count and, when `tag`
    is in event_tags, appends (tag, start, end, meta) to event_log."""
    global launch_count
    timed = event_log is not None and tag in event_tags
    if timed:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    rc = fn(*args, torch.cuda.current_stream().cuda_stream)
    if timed:
        e1.record()
    if rc:
        _lib.check(rc, fn.__name__)
    launch_count += kernels
    if timed:
        event_log.append((tag, e0, e1, meta))


def _device(t: torch.Tensor, name: str) -> int:
    """The current CUDA device, queried once per call for `_ptr`.  `t` is checked first, so a CPU tensor is refused
    before any CUDA query (and the same way on a machine without a GPU)."""
    if not t.is_cuda:
        raise _lib.AmbError(f"{name}: expected a CUDA tensor (there is no CPU fallback)")
    return torch.cuda.current_device()


def _ptr(t: Optional[torch.Tensor], dtype, name: str, dev: int) -> Optional[int]:
    """Device pointer of a tensor handed to the C ABI (None -> NULL) once it has `dtype` (or one of a tuple of dtypes)
    and lives on `dev`, the current device from `_device`."""
    if t is None:
        return None
    if t.dtype != dtype and not (type(dtype) is tuple and t.dtype in dtype):
        raise _lib.AmbError(f"{name}: expected {dtype}, got {t.dtype}")
    # the C ABI launches on the CURRENT device and stream: a tensor of another device would be an illegal access (or
    # silent peer traffic).  The module-level entry points (B200Denoiser.forward, B200SchedulerFlow.denoise, ...) make
    # their own device current; direct callers of ops must do the same.
    if t.get_device() != dev:
        if not t.is_cuda:
            raise _lib.AmbError(f"{name}: expected a CUDA tensor (there is no CPU fallback)")
        raise _lib.AmbError(f"{name}: tensor lives on {t.device} but the current device is cuda:{dev}"
                            " (wrap the call in torch.cuda.device(tensor.device))")
    return t.data_ptr()


def cfg_euler_step(latents: torch.Tensor, pred: torch.Tensor, scales: list[float], dt_signed: float,
                   frame_update: torch.Tensor, *, n_branches: int, branch_stride: int, frame_stride: int,
                   frame_offset: int, n_per_frame: int) -> None:
    """In-place x[f] += dt * (p0 + sum_i s_i (p_{i+1} - p_i)) on frames with frame_update[f] != 0.

    Replaces guidance.py:95-118 + scheduler.py:238-248 of the reference."""
    dev = _device(latents, "latents")
    arr = (C.c_float * max(1, len(scales)))(*scales)
    _launch(_abi.amb_cfg_euler_step, 1, _ptr(latents, torch.float32, "latents", dev), _ptr(pred, torch.bfloat16, "pred", dev),
            n_branches, arr, float(dt_signed), _ptr(frame_update, torch.uint8, "frame_update", dev), frame_update.numel(),
            n_per_frame, branch_stride, frame_stride, frame_offset)


def layernorm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float,
              out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Affine LayerNorm over the last dim of a 2-D (rows, cols) tensor, fp32 statistics, bf16 (default) or fp32 output."""
    dev = _device(x, "x")
    assert x.dim() == 2 and x.stride(1) == 1
    rows, cols = x.shape
    if out is None:
        out = torch.empty((rows, cols), dtype=torch.bfloat16, device=x.device)
    _launch(_abi.amb_layernorm, 1, _ptr(x, _FLOAT, "x", dev), int(x.dtype == torch.float32), x.stride(0),
            _ptr(gamma, torch.float32, "gamma", dev), _ptr(beta, torch.float32, "beta", dev), _ptr(out, _FLOAT, "out", dev),
            int(out.dtype == torch.float32), out.stride(0), rows, cols, float(eps),
            tag="layernorm", meta=(rows, cols, x.element_size() + out.element_size()))
    return out


def patchify(pixels: torch.Tensor, patch: int, kpad: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """im2col of (T,3,H,W) fp32 pixels -> (T*(H/P)*(W/P), kpad) bf16 rows for the patch-embedding GEMM."""
    dev = _device(pixels, "pixels")
    assert pixels.is_contiguous() and pixels.dim() == 4 and pixels.shape[1] == 3
    T, _, H, W = pixels.shape
    rows = T * (H // patch) * (W // patch)
    if out is None:
        out = torch.empty(rows, kpad, dtype=torch.bfloat16, device=pixels.device)
    _launch(_abi.amb_patchify, 1, _ptr(pixels, torch.float32, "pixels", dev), _ptr(out, torch.bfloat16, "out", dev),
            T, H, W, patch, kpad)
    return out


def alpha_rows(source_alpha: float, target_alpha: float, size: int, out_rows: torch.Tensor) -> None:
    """Write the (source, target) alpha token (2*size fp32 values) into every row of the strided 2-D view `out_rows`."""
    dev = _device(out_rows, "out_rows")
    assert out_rows.dim() == 2 and out_rows.shape[1] == 2 * size and out_rows.stride(1) == 1
    _launch(_abi.amb_alpha_rows, 1, float(source_alpha), float(target_alpha), size,
            _ptr(out_rows, torch.float32, "out_rows", dev), out_rows.stride(0), out_rows.shape[0])


def point_embedding(points: torch.Tensor, num_freqs: int, include_pi: bool, kpad: int) -> torch.Tensor:
    """(V, 3+E) fp32 query points -> (V, kpad) fp32 [x | sin | cos | extra | 0-pad] rows."""
    dev = _device(points, "points")
    assert points.dim() == 2 and points.is_contiguous()
    V, in_dim = points.shape
    out = torch.empty(V, kpad, dtype=torch.float32, device=points.device)
    _launch(_abi.amb_point_embedding, 1, _ptr(points, torch.float32, "points", dev), V, in_dim, in_dim - 3, num_freqs,
            int(include_pi), _ptr(out, torch.float32, "out", dev), kpad)
    return out


def split3(src: torch.Tensor, out: torch.Tensor, seg: Optional[int] = None, weight: bool = False) -> torch.Tensor:
    """fp32 (rows, cols) -> bf16 (rows, 3*cols) split operand: [hi|lo|hi] per segment (activations) or [hi|hi|lo] (weights)."""
    dev = _device(src, "src")
    assert src.dim() == 2 and out.dim() == 2 and src.stride(1) == 1 and out.stride(1) == 1
    rows, cols = src.shape
    assert out.shape[0] >= rows and out.shape[1] == 3 * cols
    _launch(_abi.amb_split3_bf16, 1, _ptr(src, torch.float32, "src", dev), src.stride(0), rows, cols, seg or cols,
            int(weight), _ptr(out, torch.bfloat16, "out", dev), out.stride(0))
    return out


def softmax_split3(scores: torch.Tensor, n: int, scale: float, out: torch.Tensor) -> torch.Tensor:
    """Row softmax over the first n columns of fp32 `scores` (rows, n_pad), written as [P_hi|P_lo|P_hi] (rows, 3*n_pad)."""
    dev = _device(scores, "scores")
    rows, n_pad = scores.shape
    assert scores.stride(1) == 1 and out.stride(1) == 1 and out.shape == (rows, 3 * n_pad)
    _launch(_abi.amb_softmax_split3, 1, _ptr(scores, torch.float32, "scores", dev), scores.stride(0), rows, n, n_pad,
            float(scale), _ptr(out, torch.bfloat16, "out", dev), out.stride(0))
    return out


def displacement_out(logits: torch.Tensor, out_dim: int, out: torch.Tensor) -> torch.Tensor:
    dev = _device(logits, "logits")
    assert logits.dim() == 2 and logits.stride(1) == 1 and out.is_contiguous()
    _launch(_abi.amb_displacement_out, 1, _ptr(logits, torch.float32, "logits", dev), logits.stride(0), logits.shape[0],
            out_dim, _ptr(out, torch.float32, "out", dev))
    return out


def resize_h_u8(src: torch.Tensor, y0: int, n_rows: int, bounds: torch.Tensor, coeffs: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """Horizontal pass of Pillow's uint8 resample on source rows [y0, y0+n_rows): src (n, H, W, 3|4) u8 -> out (n, n_rows, out_w, 3)."""
    dev = _device(src, "src")
    assert src.dim() == 4 and src.is_contiguous() and out.is_contiguous() and bounds.is_contiguous() and coeffs.is_contiguous()
    n, H, W, cin = src.shape
    out_w, ksize = coeffs.shape
    assert out.shape == (n, n_rows, out_w, 3) and bounds.shape == (out_w, 2)
    _launch(_abi.amb_resize_h_u8, 1, _ptr(src, torch.uint8, "src", dev), n, H, W, cin, y0, n_rows,
            _ptr(bounds, torch.int32, "bounds", dev), _ptr(coeffs, torch.int32, "coeffs", dev), ksize, out_w,
            _ptr(out, torch.uint8, "out", dev))
    return out


def resize_v_normalize(src: torch.Tensor, y0: int, bounds: torch.Tensor, coeffs: torch.Tensor, lut: torch.Tensor, mean, std,
                       out: torch.Tensor, out_u8: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Vertical pass + 1/255 rescale (lut) + mean/std + CHW: src (n, n_rows, out_w, 3) u8 -> out (n, 3, out_h, out_w) fp32."""
    dev = _device(src, "src")
    assert src.is_contiguous() and out.is_contiguous() and lut.numel() == 256
    n, n_rows, out_w, _ = src.shape
    out_h, ksize = coeffs.shape
    assert out.shape == (n, 3, out_h, out_w) and bounds.shape == (out_h, 2)
    if out_u8 is not None:
        assert out_u8.shape == (n, out_h, out_w, 3) and out_u8.is_contiguous()
    m = (C.c_float * 3)(*[float(v) for v in mean])
    s = (C.c_float * 3)(*[float(v) for v in std])
    _launch(_abi.amb_resize_v_normalize, 1, _ptr(src, torch.uint8, "src", dev), n, n_rows, y0, out_w,
            _ptr(bounds, torch.int32, "bounds", dev), _ptr(coeffs, torch.int32, "coeffs", dev), ksize, out_h,
            _ptr(lut, torch.float32, "lut", dev), m, s, _ptr(out, torch.float32, "out", dev),
            _ptr(out_u8, torch.uint8, "out_u8", dev))
    return out


def alpha_stats(rgba: torch.Tensor) -> torch.Tensor:
    """(n, H, W, 4) u8 RGBA frames -> (n, 5) int32: xmin, ymin, xmax, ymax of alpha > 0 and the count of alpha > 127."""
    dev = _device(rgba, "rgba")
    assert rgba.dim() == 4 and rgba.shape[3] == 4 and rgba.is_contiguous()
    n, H, W, _ = rgba.shape
    stats = torch.empty(n, 5, dtype=torch.int32, device=rgba.device)
    _launch(_abi.amb_alpha_stats, 2, _ptr(rgba, torch.uint8, "rgba", dev), n, H, W, _ptr(stats, torch.int32, "stats", dev))
    return stats


def composite_crop_pad(rgba: torch.Tensor, box: tuple, pad_x: int, pad_y: int) -> torch.Tensor:
    """RGBA frames -> white-composited, cropped to box = (x, y, w, h), padded uint8 RGB frames (n, h + 2 pad_y, w + 2 pad_x, 3)."""
    dev = _device(rgba, "rgba")
    assert rgba.dim() == 4 and rgba.shape[3] == 4 and rgba.is_contiguous()
    n, H, W, _ = rgba.shape
    x, y, w, h = (int(v) for v in box)
    out = torch.empty(n, h + 2 * pad_y, w + 2 * pad_x, 3, dtype=torch.uint8, device=rgba.device)
    _launch(_abi.amb_composite_crop_pad, 1, _ptr(rgba, torch.uint8, "rgba", dev), n, H, W, x, y, w, h, int(pad_x), int(pad_y),
            _ptr(out, torch.uint8, "out", dev))
    return out


def nearest_neighbors(query: torch.Tensor, reference: torch.Tensor, want_index: bool = True):
    """(Q, 3), (R, 3) fp32 CUDA points -> (distance (Q,) fp32, index (Q,) int32) of each query's nearest reference point."""
    dev = _device(query, "query")
    assert query.dim() == 2 and query.shape[1] == 3 and reference.dim() == 2 and reference.shape[1] == 3
    q, r = query.contiguous(), reference.contiguous()
    dist = torch.empty(q.shape[0], dtype=torch.float32, device=q.device)
    idx = torch.empty(q.shape[0], dtype=torch.int32, device=q.device) if want_index else None
    scratch = torch.empty(q.shape[0], dtype=torch.int64, device=q.device)
    _launch(_abi.amb_nearest_neighbors, 3, _ptr(q, torch.float32, "query", dev), q.shape[0],
            _ptr(r, torch.float32, "reference", dev), r.shape[0], _ptr(scratch, torch.int64, "scratch", dev),
            _ptr(dist, torch.float32, "dist", dev), _ptr(idx, torch.int32, "idx", dev))
    return dist, idx


def cast_bf16(src: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    dev = _device(src, "src")
    assert src.is_contiguous()
    if out is None:
        out = torch.empty(src.shape, dtype=torch.bfloat16, device=src.device)
    _launch(_abi.amb_cast_f32_bf16, 1, _ptr(src, torch.float32, "src", dev), _ptr(out, torch.bfloat16, "out", dev),
            src.numel())
    return out


def timestep_embedding(t: torch.Tensor, channels: int, out: Optional[torch.Tensor] = None, *,
                       mask: Optional[torch.Tensor] = None, rows: Optional[int] = None) -> torch.Tensor:
    """Row r: sinusoidal embedding of t[r % len(t)] * (1 - mask[r]) (temporal_denoiser.py:209-213)."""
    dev = _device(t, "t")
    if mask is not None:
        rows = mask.numel()
    if rows is None:
        rows = t.numel()
    if out is None:
        out = torch.empty((rows, channels), dtype=torch.bfloat16, device=t.device)
    _launch(_abi.amb_timestep_embedding, 1, _ptr(t, torch.float32, "t", dev), t.numel(), _ptr(mask, torch.float32, "mask", dev),
            rows, channels, _ptr(out, torch.bfloat16, "out", dev))
    return out


def add_bias_rows(y: torch.Tensor, bias: torch.Tensor) -> None:
    dev = _device(y, "y")
    assert y.dim() == 2 and y.stride(1) == 1
    _launch(_abi.amb_add_bias_rows, 1, _ptr(y, _FLOAT, "y", dev), int(y.dtype == torch.float32), y.stride(0),
            _ptr(bias, torch.float32, "bias", dev), y.shape[0], y.shape[1])


def gemm(a: torch.Tensor, w: torch.Tensor, out: torch.Tensor, *, bias: Optional[torch.Tensor] = None,
         a2: Optional[torch.Tensor] = None, residual: Optional[torch.Tensor] = None, act: int = 0,
         col_scale: Optional[torch.Tensor] = None, row_map: Optional[tuple[int, int, int]] = None,
         norm: Optional[dict] = None, out2: Optional[torch.Tensor] = None, tag: str = "gemm") -> torch.Tensor:
    """out = epilogue(cat[a, a2] @ w.T).  a:(m,k1) bf16, a2:(m,k2) bf16 or None, w:(n,k1+k2) bf16, out bf16/fp32.

    norm = dict(cols=, seg=, w0=, w1=, eps=, rope_cols=, cos=, sin=, rows_per_pos=) enables the per-head
    RMSNorm(+RoPE) epilogue of attention_processor.py:106-130."""
    dev = _device(a, "a")
    assert a.dim() == 2 and w.dim() == 2 and out.dim() == 2
    assert a.stride(1) == 1 and w.stride(1) == 1 and out.stride(1) == 1
    g = _lib.GemmArgs()  # zero-initialised: every unused pointer is NULL, every unused size 0
    m, k1 = a.shape
    n, k = w.shape
    g.a, g.lda = _ptr(a, torch.bfloat16, "a", dev), a.stride(0)
    if a2 is not None:
        assert a2.shape[0] == m and a2.stride(1) == 1 and k1 + a2.shape[1] == k
        g.a2, g.lda2, g.k_split = _ptr(a2, torch.bfloat16, "a2", dev), a2.stride(0), k1
    else:
        assert k1 == k, f"a has k={k1}, w has k={k}"
    g.w, g.ldw = _ptr(w, torch.bfloat16, "w", dev), w.stride(0)
    g.c, g.ldc, g.c_fp32 = _ptr(out, _FLOAT, "out", dev), out.stride(0), int(out.dtype == torch.float32)
    g.m, g.n, g.k = m, n, k
    if out2 is not None:  # bf16 copy of the result (GEMM operand of a later linear)
        assert out2.shape == out.shape and out2.stride(1) == 1
        g.c2, g.ldc2 = _ptr(out2, torch.bfloat16, "out2", dev), out2.stride(0)
    g.bias = _ptr(bias, torch.float32, "bias", dev)
    if residual is not None:
        assert residual.stride(1) == 1
        g.residual, g.ldr = _ptr(residual, _FLOAT, "residual", dev), residual.stride(0)
        g.res_fp32 = int(residual.dtype == torch.float32)
    g.act = act
    g.col_scale = _ptr(col_scale, torch.float32, "col_scale", dev)
    if row_map is not None:
        g.grp_rows, g.grp_stride, g.row_off = row_map
    if norm is None:
        g.rope_rows_per_pos = 1
    else:
        g.norm_cols, g.norm_seg = norm.get("cols", 0), norm.get("seg", norm.get("cols", 0))
        g.norm_w0 = _ptr(norm.get("w0"), torch.float32, "norm w0", dev)
        g.norm_w1 = _ptr(norm.get("w1"), torch.float32, "norm w1", dev)
        g.norm_eps = float(norm.get("eps", 0.0))
        g.rope_cols = norm.get("rope_cols", 0)
        g.rope_cos = _ptr(norm.get("cos"), torch.float32, "rope cos", dev)
        g.rope_sin = _ptr(norm.get("sin"), torch.float32, "rope sin", dev)
        g.rope_rows_per_pos = norm.get("rows_per_pos", 1)
    _launch(_abi.amb_gemm_bf16, 1, C.byref(g), tag=tag, meta=(m, n, k))
    return out


def attn_small_f32(qkv: torch.Tensor, frames: int, seq: int, heads: int, scale: float, out: torch.Tensor,
                   tag: str = "attn_small") -> torch.Tensor:
    """fp32 attention of `frames` independent sequences of `seq` <= 320 tokens, head_dim 64 (DinoV2).
    qkv: fp32 (frames * seq, 3 * heads * 64) = [q | k | v] of a fused projection; out: fp32 (frames * seq, heads * 64)."""
    dev = _device(qkv, "qkv")
    D = heads * 64
    assert qkv.dim() == 2 and out.dim() == 2 and qkv.stride(1) == 1 and out.stride(1) == 1
    assert qkv.shape == (frames * seq, 3 * D) and out.shape == (frames * seq, D)
    base = _ptr(qkv, torch.float32, "qkv", dev)
    _launch(_abi.amb_attn_small_f32, 1, base, base + 4 * D, base + 8 * D, qkv.stride(0), frames, seq, heads, float(scale),
            _ptr(out, torch.float32, "out", dev), out.stride(0), tag=tag, meta=(frames, heads, seq, seq, 64))
    return out


def flash_attn(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, out: torch.Tensor, scale: float, *,
               kv_chunks: int = 1, tag: str = "attn") -> torch.Tensor:
    """softmax(scale q kᵀ) v, non-causal.  q:(B,Sq,H,D) k,v:(B,Sk,H,D) out:(B,Sq,H,D) — arbitrary (16-byte aligned)
    strides with unit stride on D, so views into a fused QKV buffer work in place.

    With kv_chunks > 1, k/v are (B, chunks, Sk_chunk, H, D) (rank-c all-gathered K/V of the frame-sharded window)."""
    dev = _device(q, "q")
    assert q.stride(-1) == 1 and k.stride(-1) == 1 and v.stride(-1) == 1 and out.stride(-1) == 1
    a = _lib.AttnArgs()
    B, Sq, H, D = q.shape
    a.q, a.k = _ptr(q, torch.bfloat16, "q", dev), _ptr(k, torch.bfloat16, "k", dev)
    a.v, a.o = _ptr(v, torch.bfloat16, "v", dev), _ptr(out, torch.bfloat16, "out", dev)
    a.q_stride_b, a.q_stride_s, a.q_stride_h = q.stride(0), q.stride(1), q.stride(2)
    a.o_stride_b, a.o_stride_s, a.o_stride_h = out.stride(0), out.stride(1), out.stride(2)
    if kv_chunks > 1:
        assert k.dim() == 5 and v.dim() == 5 and k.shape[1] == kv_chunks
        a.k_stride_b, a.k_chunk_stride, a.k_stride_s, a.k_stride_h = k.stride(0), k.stride(1), k.stride(2), k.stride(3)
        a.v_stride_b, a.v_chunk_stride, a.v_stride_s, a.v_stride_h = v.stride(0), v.stride(1), v.stride(2), v.stride(3)
        a.sk_chunk = k.shape[2]
        a.sk = k.shape[1] * k.shape[2]
    else:
        assert k.dim() == 4 and v.dim() == 4
        a.k_stride_b, a.k_stride_s, a.k_stride_h = k.stride(0), k.stride(1), k.stride(2)
        a.v_stride_b, a.v_stride_s, a.v_stride_h = v.stride(0), v.stride(1), v.stride(2)
        a.sk_chunk = k.shape[1]
        a.sk = k.shape[1]
    a.kv_chunks = kv_chunks
    a.batch, a.heads, a.sq, a.head_dim = B, H, Sq, D
    a.scale = float(scale)
    _launch(_abi.amb_flash_attn_fwd, 1, C.byref(a), tag=tag, meta=(B, H, Sq, a.sk, D))
    return out


# ---- Stage 0's anchor mesh: octree refinement + dual marching cubes (csrc/geometry.cu) --------------------------------------
def _scan_scratch(n_items: int, device) -> torch.Tensor:
    return torch.empty(_lib.scan_scratch_ints(n_items), dtype=torch.int32, device=device)


def _cube(t: torch.Tensor, name: str) -> int:
    assert t.dim() == 3 and t.shape[0] == t.shape[1] == t.shape[2] and t.is_contiguous(), f"{name}: expected a contiguous cube"
    return t.shape[0]


def octree_near_surface(grid: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """(n,n,n) fp32 logits -> uint8 mask of the near-surface band (sign change to a face neighbour, or |logit| < 0.95)."""
    dev = _device(grid, "grid")
    n = _cube(grid, "grid")
    out = torch.empty_like(grid, dtype=torch.uint8) if out is None else out
    _cube(out, "out")
    _launch(_abi.amb_octree_near_surface, 1, _ptr(grid, torch.float32, "grid", dev), n, _ptr(out, torch.uint8, "out", dev))
    return out


def octree_dilate(mask: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """3x3x3 zero-padded dilation of a uint8 mask (out must not alias mask)."""
    dev = _device(mask, "mask")
    n = _cube(mask, "mask")
    out = torch.empty_like(mask) if out is None else out
    _cube(out, "out")
    _launch(_abi.amb_octree_dilate, 1, _ptr(mask, torch.uint8, "mask", dev), n, _ptr(out, torch.uint8, "out", dev))
    return out


def octree_mark_upsampled(mask: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """(n,n,n) uint8 -> (2n-1)^3 uint8 with fine[2x, 2y, 2z] = (mask[x, y, z] != 0) and zeros elsewhere."""
    dev = _device(mask, "mask")
    n = _cube(mask, "mask")
    fine = torch.empty((2 * n - 1,) * 3, dtype=torch.uint8, device=mask.device) if out is None else out
    assert _cube(fine, "out") == 2 * n - 1, "out: expected a (2n-1)^3 cube"
    _launch(_abi.amb_octree_mark_upsampled, 2, _ptr(mask, torch.uint8, "mask", dev), n, _ptr(fine, torch.uint8, "fine", dev))
    return fine


def octree_points(mask: torch.Tensor, resolution, bbox_min) -> tuple[torch.Tensor, torch.Tensor]:
    """Set cells of a uint8 mask in grid order -> (xyz (P, 3) fp32 = fp32(idx) * resolution + bbox_min, linear index (P,) int32).
    Reads P back to the host (one sync)."""
    dev = _device(mask, "mask")
    n = _cube(mask, "mask")
    scratch = _scan_scratch(n ** 3, mask.device)
    # the count call carries all 4 of the wrapper's kernels, so the total is the same when no point is emitted
    _launch(_abi.amb_octree_count_points, 4, _ptr(mask, torch.uint8, "mask", dev), n, _ptr(scratch, torch.int32, "scratch", dev))
    count = int(scratch[-1].item())
    xyz = torch.empty(count, 3, dtype=torch.float32, device=mask.device)
    index = torch.empty(count, dtype=torch.int32, device=mask.device)
    res = (C.c_float * 3)(*[float(v) for v in resolution])
    lo = (C.c_float * 3)(*[float(v) for v in bbox_min])
    if count:
        _launch(_abi.amb_octree_emit_points, 0, _ptr(mask, torch.uint8, "mask", dev), n,
                _ptr(scratch, torch.int32, "scratch", dev), res, lo, _ptr(xyz, torch.float32, "xyz", dev),
                _ptr(index, torch.int32, "index", dev))
    return xyz, index


def grid_fill(grid: torch.Tensor, value: float) -> torch.Tensor:
    dev = _device(grid, "grid")
    assert grid.is_contiguous()
    _launch(_abi.amb_grid_fill, 1, _ptr(grid, torch.float32, "grid", dev), grid.numel(), float(value))
    return grid


def grid_replace(grid: torch.Tensor, value_from: float, value_to: float) -> torch.Tensor:
    dev = _device(grid, "grid")
    assert grid.is_contiguous()
    _launch(_abi.amb_grid_replace, 1, _ptr(grid, torch.float32, "grid", dev), grid.numel(), float(value_from), float(value_to))
    return grid


def grid_scatter(values: torch.Tensor, index: torch.Tensor, grid: torch.Tensor) -> torch.Tensor:
    """grid.view(-1)[index[i]] = values[i, 0] for fp32 `values` (P, k) with any row stride."""
    dev = _device(values, "values")
    assert values.dim() == 2 and values.shape[0] == index.numel() and index.is_contiguous() and grid.is_contiguous()
    _launch(_abi.amb_grid_scatter, 1, _ptr(values, torch.float32, "values", dev), values.stride(0),
            _ptr(index, torch.int32, "index", dev), index.numel(), _ptr(grid, torch.float32, "grid", dev))
    return grid


def dual_marching_cubes(grid: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """Dual marching cubes of the zero level set of an (n,n,n) fp32 grid (inside = value > 0; non-finite cells emit nothing)
    -> vertices (V, 3) fp32 in grid-index units, faces (F, 3) int32 wound outward.  Reads V and F back (one sync)."""
    dev = _device(grid, "grid")
    n = _cube(grid, "grid")
    cases = torch.empty((n - 1,) * 3, dtype=torch.uint8, device=grid.device)
    vs, fs = _scan_scratch((n - 1) ** 3, grid.device), _scan_scratch(n ** 3, grid.device)
    common = (_ptr(grid, torch.float32, "grid", dev), n, _ptr(cases, torch.uint8, "cases", dev),
              _ptr(vs, torch.int32, "vertex scratch", dev), _ptr(fs, torch.int32, "face scratch", dev))
    _launch(_abi.amb_dmc_count, 9, *common)  # the 9 kernels of both calls
    nv, nf = (int(v) for v in torch.stack([vs[-1], fs[-1]]).tolist())
    voff = torch.empty((n - 1,) * 3, dtype=torch.int32, device=grid.device)
    verts = torch.empty(max(nv, 1), 3, dtype=torch.float32, device=grid.device)
    faces = torch.empty(max(nf, 1), 3, dtype=torch.int32, device=grid.device)
    _launch(_abi.amb_dmc_emit, 0, *common, _ptr(voff, torch.int32, "vertex offsets", dev),
            _ptr(verts, torch.float32, "vertices", dev), _ptr(faces, torch.int32, "faces", dev))
    return verts[:nv], faces[:nf]


# ---- mesh input: the TripoSG VAE encoder's point sampling and posterior (csrc/point_sampling.cu) ---------------------------
FPS_MAX_POINTS = 16384


def farthest_point_sample(points_xyz_view: torch.Tensor, k: int, start) -> torch.Tensor:
    """Farthest-point sampling of (B, N, >=3) fp32 points (any row and batch stride: the xyz of (B, N, 6) surface rows are
    read in place) -> (B, k) int64 indices, the first of each row `start[b]`; ties go to the lowest index.  `start`: (B,)
    int64 on the host (range-checked) or on the device (caller's guarantee).  N <= 16384."""
    dev = _device(points_xyz_view, "points")
    p = points_xyz_view
    assert p.dim() == 3 and p.shape[2] >= 3 and p.stride(2) == 1
    B, N = p.shape[0], p.shape[1]
    start = torch.as_tensor(start, dtype=torch.int64).reshape(-1)
    if start.numel() != B:
        raise _lib.AmbError(f"farthest_point_sample: {start.numel()} start indices for a batch of {B}")
    if not start.is_cuda:
        if B and (int(start.min()) < 0 or int(start.max()) >= N):
            raise _lib.AmbError(f"farthest_point_sample: start index outside [0, {N})")
        start = start.to(p.device)
    out = torch.empty(B, int(k), dtype=torch.int64, device=p.device)
    _launch(_abi.amb_farthest_point_sample, 1, _ptr(p, torch.float32, "points", dev), B, N, p.stride(1),
            p.stride(0) if B > 1 else N * p.stride(1), _ptr(start.contiguous(), torch.int64, "start", dev), int(k),
            _ptr(out, torch.int64, "out", dev), tag="fps", meta=(B, N, int(k)))
    return out


def gaussian_sample(params: torch.Tensor, eps: Optional[torch.Tensor] = None, *, z: Optional[torch.Tensor] = None,
                    logvar: Optional[torch.Tensor] = None, std: Optional[torch.Tensor] = None) -> Optional[torch.Tensor]:
    """DiagonalGaussianDistribution on fp32 `params` (rows, >= 2C) (any row stride; C from the outputs' width):
    logvar = clamp(params[:, C:2C], -30, 20), std = exp(0.5 logvar), z = params[:, :C] + std * eps.  Writes whichever of
    z / logvar / std is given (contiguous (rows, C) fp32); with `eps` and no `z`, allocates and returns z."""
    dev = _device(params, "params")
    assert params.dim() == 2 and params.stride(1) == 1
    rows = params.shape[0]
    if eps is not None and z is None:
        z = torch.empty(eps.shape, dtype=torch.float32, device=params.device)
    outs = [t for t in (z, logvar, std) if t is not None]
    if not outs:
        raise _lib.AmbError("gaussian_sample: nothing to write")
    C_ = outs[0].shape[-1]
    for t, nme in ((z, "z"), (logvar, "logvar"), (std, "std"), (eps, "eps")):
        if t is not None:
            assert t.is_contiguous() and t.numel() == rows * C_, f"{nme}: expected {rows} x {C_} contiguous values"
    if params.shape[1] < 2 * C_:
        raise _lib.AmbError(f"gaussian_sample: params have {params.shape[1]} columns, need {2 * C_}")
    _launch(_abi.amb_gaussian_sample, 1, _ptr(params, torch.float32, "params", dev), params.stride(0), rows, C_,
            _ptr(eps, torch.float32, "eps", dev), _ptr(z, torch.float32, "z", dev),
            _ptr(logvar, torch.float32, "logvar", dev), _ptr(std, torch.float32, "std", dev))
    return z


# ---- anchor-mesh post-processing: quadric edge-collapse decimation and floater removal (csrc/mesh_process.cu) -------------
NO_KEY = (1 << 64) - 1


def mesh_scan_scratch(n_vertices: int, n_faces: int, device) -> tuple[torch.Tensor, torch.Tensor]:
    """(work (V,) int32, scan scratch for max(V, F) items) shared by the mesh_* calls on one mesh."""
    return torch.empty(max(n_vertices, 1), dtype=torch.int32, device=device), _scan_scratch(max(n_vertices, n_faces), device)


def _scan_total(scan: torch.Tensor, n_items: int) -> int:
    return int(scan[_lib.scan_scratch_ints(n_items) - 1].item())


def _mesh_faces(faces: torch.Tensor) -> int:
    assert faces.dim() == 2 and faces.shape[1] == 3 and faces.is_contiguous(), "faces: expected a contiguous (F, 3) tensor"
    return faces.shape[0]


def _adjacency(adjacency, dev: int) -> tuple:
    """Pointers of mesh_adjacency's (vf_offsets, vf_faces, neighbours)."""
    return tuple(_ptr(t, torch.int32, nme, dev) for t, nme in zip(adjacency[:3], ("vf_offsets", "vf_faces", "neighbours")))


def mesh_adjacency(faces: torch.Tensor, n_vertices: int, work: torch.Tensor, scan: torch.Tensor):
    """Vertex -> face CSR of (F, 3) int32 faces (F >= 1) and the edge list -> (vf_offsets (V+1), vf_faces (3F), neighbours (6F),
    edges (E, 5) int32 = a < b, face count, f0, f1 ordered by (a, b), flags (V) uint8: 1 boundary, 2 non-manifold).
    Reads E back (one sync)."""
    dev = _device(faces, "faces")
    F = _mesh_faces(faces)
    off = torch.empty(n_vertices + 1, dtype=torch.int32, device=faces.device)
    vf = torch.empty(3 * F, dtype=torch.int32, device=faces.device)
    nb = torch.empty(6 * F, dtype=torch.int32, device=faces.device)
    fp, adj = _ptr(faces, torch.int32, "faces", dev), _adjacency((off, vf, nb), dev)
    wp, sp = _ptr(work, torch.int32, "work", dev), _ptr(scan, torch.int32, "scan", dev)
    _launch(_abi.amb_mesh_adjacency, 14, fp, F, n_vertices, wp, sp, *adj)  # the 14 kernels of both calls
    E = _scan_total(scan, n_vertices)
    edges = torch.empty(max(E, 1), 5, dtype=torch.int32, device=faces.device)
    flags = torch.empty(max(n_vertices, 1), dtype=torch.uint8, device=faces.device)
    _launch(_abi.amb_mesh_edges, 0, fp, F, n_vertices, *adj, wp, sp, _ptr(edges, torch.int32, "edges", dev),
            _ptr(flags, torch.uint8, "flags", dev))
    return off, vf, nb, edges[:E], flags


def mesh_quadrics(positions: torch.Tensor, faces: torch.Tensor, adjacency) -> torch.Tensor:
    """(V, 10) fp64 initial error quadrics: area-weighted face planes plus weighted boundary-edge planes."""
    dev = _device(positions, "positions")
    _mesh_faces(faces)
    V = positions.shape[0]
    q = torch.empty(V, 10, dtype=torch.float64, device=positions.device)
    _launch(_abi.amb_mesh_quadrics, 1, _ptr(positions, torch.float64, "positions", dev), _ptr(faces, torch.int32, "faces", dev),
            V, *_adjacency(adjacency, dev), _ptr(q, torch.float64, "quadrics", dev))
    return q


def mesh_collapse_select(positions: torch.Tensor, quadrics: torch.Tensor, faces: torch.Tensor, adjacency):
    """One round's independent set of cheapest valid collapses -> dict(keys (E,), targets (E, 3), vertex_min (2V,),
    remap (V,), winners (n, 2) = (key, face count) unordered, removed = faces the winners remove).  Keys are uint64 bit
    patterns held in int64 tensors.  Reads the winner count back (one sync)."""
    dev = _device(positions, "positions")
    edges, flags = adjacency[3:]
    V, E, d = positions.shape[0], edges.shape[0], positions.device
    keys = torch.empty(max(E, 1), dtype=torch.int64, device=d)
    targets = torch.empty(max(E, 1), 3, dtype=torch.float64, device=d)
    vmin = torch.empty(2 * V, dtype=torch.int64, device=d)
    remap = torch.empty(V, dtype=torch.int32, device=d)
    counters = torch.empty(2, dtype=torch.int64, device=d)
    winners = torch.empty(max(E, 1), 2, dtype=torch.int64, device=d)
    _launch(_abi.amb_mesh_collapse_select, 5, _ptr(positions, torch.float64, "positions", dev),
            _ptr(quadrics, torch.float64, "quadrics", dev), _ptr(faces, torch.int32, "faces", dev), V,
            *_adjacency(adjacency, dev), _ptr(edges, torch.int32, "edges", dev), E, _ptr(flags, torch.uint8, "flags", dev),
            _ptr(keys, torch.int64, "keys", dev), _ptr(targets, torch.float64, "targets", dev),
            _ptr(vmin, torch.int64, "vertex_min", dev), _ptr(remap, torch.int32, "remap", dev),
            _ptr(counters, torch.int64, "counters", dev), _ptr(winners, torch.int64, "winners", dev))
    n_win, removed = (int(v) for v in counters.tolist())
    return dict(keys=keys, targets=targets, vertex_min=vmin, remap=remap, winners=winners[:n_win], removed=removed)


def mesh_collapse_apply(edges: torch.Tensor, selection: dict, key_limit: int, positions: torch.Tensor,
                        quadrics: torch.Tensor) -> torch.Tensor:
    """Collapse every winner of `selection` whose key <= key_limit (b into a, a to its target, Q_a += Q_b), in place ->
    the round's remap (V,) int32."""
    dev = _device(positions, "positions")
    s = selection
    _launch(_abi.amb_mesh_collapse_apply, 1, _ptr(edges, torch.int32, "edges", dev), edges.shape[0], positions.shape[0],
            _ptr(s["keys"], torch.int64, "keys", dev), _ptr(s["targets"], torch.float64, "targets", dev),
            _ptr(s["vertex_min"], torch.int64, "vertex_min", dev), int(key_limit), _ptr(s["remap"], torch.int32, "remap", dev),
            _ptr(positions, torch.float64, "positions", dev), _ptr(quadrics, torch.float64, "quadrics", dev))
    return s["remap"]


def mesh_compact_faces(faces: torch.Tensor, scan: torch.Tensor, *, remap: Optional[torch.Tensor] = None,
                       labels: Optional[torch.Tensor] = None, sizes: Optional[torch.Tensor] = None,
                       min_size: int = 0) -> torch.Tensor:
    """The faces, in order, whose corners (through `remap`) are distinct and, with `labels`, whose component has >= min_size
    faces (`sizes[labels[f]]`) -> (F', 3) int32.  Reads F' back (one sync)."""
    dev = _device(faces, "faces")
    F = _mesh_faces(faces)
    out = torch.empty(max(F, 1), 3, dtype=torch.int32, device=faces.device)
    _launch(_abi.amb_mesh_compact_faces, 3, _ptr(faces, torch.int32, "faces", dev), F, _ptr(remap, torch.int32, "remap", dev),
            _ptr(labels, torch.int32, "labels", dev), _ptr(sizes, torch.int32, "sizes", dev), int(min_size),
            _ptr(scan, torch.int32, "scan", dev), _ptr(out, torch.int32, "out", dev))
    return out[:_scan_total(scan, F) if F else 0]


def mesh_compact_vertices(positions: torch.Tensor, faces: torch.Tensor, work: torch.Tensor,
                          scan: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """Drop unreferenced vertices, keeping the others in index order -> (positions (V', 3) fp64, faces renumbered).
    Reads V' back (one sync)."""
    dev = _device(positions, "positions")
    F = _mesh_faces(faces)
    V = positions.shape[0]
    out_p = torch.empty(max(V, 1), 3, dtype=torch.float64, device=positions.device)
    out_f = torch.empty(max(F, 1), 3, dtype=torch.int32, device=positions.device)
    _launch(_abi.amb_mesh_compact_vertices, 5, _ptr(positions, torch.float64, "positions", dev), V,
            _ptr(faces, torch.int32, "faces", dev), F, _ptr(work, torch.int32, "work", dev), _ptr(scan, torch.int32, "scan", dev),
            _ptr(out_p, torch.float64, "out positions", dev), _ptr(out_f, torch.int32, "out faces", dev))
    return out_p[:_scan_total(scan, V) if V else 0], out_f[:F]


def mesh_face_components(edges: torch.Tensor, n_faces: int) -> tuple[torch.Tensor, torch.Tensor]:
    """Components of faces joined through edges held by exactly 2 faces -> (labels (F,) int32 = the smallest face index of
    each face's component, sizes (F,) int32 = faces per label).  Union passes until stable (one sync each)."""
    dev = _device(edges, "edges")
    labels = torch.empty(max(n_faces, 1), dtype=torch.int32, device=edges.device)
    changed = torch.empty(1, dtype=torch.int32, device=edges.device)
    ep, lp = _ptr(edges, torch.int32, "edges", dev), _ptr(labels, torch.int32, "labels", dev)
    first = 1
    while True:
        _launch(_abi.amb_mesh_components, 3, ep, edges.shape[0], n_faces, first, lp, _ptr(changed, torch.int32, "changed", dev))
        first = 0
        if not int(changed.item()):
            break
    sizes = torch.empty_like(labels)
    _launch(_abi.amb_mesh_component_sizes, 2, lp, n_faces, _ptr(sizes, torch.int32, "sizes", dev))
    return labels[:n_faces], sizes[:n_faces]


# ---- multi-view normal rendering (csrc/render.cu) ----------------------------------------------------------------------------
def _render_mesh(vertices: torch.Tensor, faces: torch.Tensor) -> tuple[int, int, int]:
    """(current device, V, F) of a contiguous (V, 3) fp32 / (F, 3) int32 mesh."""
    dev = _device(vertices, "vertices")
    assert vertices.dim() == 2 and vertices.shape[1] == 3 and vertices.is_contiguous(), "vertices: expected a contiguous (V, 3) tensor"
    return dev, vertices.shape[0], _mesh_faces(faces)


def _cameras(cameras: torch.Tensor) -> int:
    assert cameras.dim() == 2 and cameras.shape[1] == 12 and cameras.is_contiguous(), "cameras: expected a contiguous (C, 12) tensor"
    return cameras.shape[0]


def vertex_normals(vertices: torch.Tensor, faces: torch.Tensor) -> torch.Tensor:
    """(V, 3) fp32 unit vertex normals: each vertex's sum of cross(v1 - v0, v2 - v0) over its faces in ascending face order,
    over max(|n|, 1e-6).  Faces need three distinct corners (the vertex -> face lists come from amb_mesh_adjacency)."""
    dev, V, F = _render_mesh(vertices, faces)
    normals = torch.empty(V, 3, dtype=torch.float32, device=vertices.device)
    if not F:
        return normals.zero_()
    work, scan = mesh_scan_scratch(V, F, vertices.device)
    off = torch.empty(V + 1, dtype=torch.int32, device=vertices.device)
    vf = torch.empty(3 * F, dtype=torch.int32, device=vertices.device)
    nb = torch.empty(6 * F, dtype=torch.int32, device=vertices.device)
    fp, adj = _ptr(faces, torch.int32, "faces", dev), _adjacency((off, vf, nb), dev)
    _launch(_abi.amb_mesh_adjacency, 11, fp, F, V, _ptr(work, torch.int32, "work", dev), _ptr(scan, torch.int32, "scan", dev),
            *adj)
    _launch(_abi.amb_render_vertex_normals, 1, _ptr(vertices, torch.float32, "vertices", dev), V, fp, *adj[:2],
            _ptr(normals, torch.float32, "normals", dev))
    return normals


def rasterize(vertices: torch.Tensor, faces: torch.Tensor, cameras: torch.Tensor, focal: float,
              image_size: int) -> torch.Tensor:
    """pix_to_face (C, 2S, 2S) int32 of the mesh seen by the (C, 12) cameras (R row-major, then T) at 2S x 2S samples: the
    face with the smallest non-negative depth at each sample, ties to the lower index, -1 where none covers it."""
    dev, V, F = _render_mesh(vertices, faces)
    n_cams, n2 = _cameras(cameras), 2 * int(image_size)
    d = vertices.device
    keys = torch.empty(max(n_cams * n2 * n2, 1), dtype=torch.int64, device=d)
    queue = torch.empty(n_cams * F + 1, dtype=torch.int32, device=d)
    pix_to_face = torch.empty(n_cams, n2, n2, dtype=torch.int32, device=d)
    _launch(_abi.amb_render_rasterize, 5 if F else 2, _ptr(vertices, torch.float32, "vertices", dev), V,
            _ptr(faces, torch.int32, "faces", dev), F, _ptr(cameras, torch.float32, "cameras", dev), n_cams, float(focal),
            int(image_size), _ptr(keys, torch.int64, "depth keys", dev), _ptr(queue, torch.int32, "queue", dev),
            _ptr(pix_to_face, torch.int32, "pix_to_face", dev))
    return pix_to_face


def shade_normals(vertices: torch.Tensor, faces: torch.Tensor, normals: torch.Tensor, cameras: torch.Tensor, focal: float,
                  pix_to_face: torch.Tensor, out: Optional[torch.Tensor] = None, column: int = 0) -> torch.Tensor:
    """The composited normal images of `rasterize`'s views as uint8 RGB, view c written to the S x S cell at column
    `column + c` of `out` (S, n_cols * S, 3) (allocated as (S, C * S, 3) when None) -> out."""
    dev, V, F = _render_mesh(vertices, faces)
    n_cams = _cameras(cameras)
    assert pix_to_face.dim() == 3 and pix_to_face.shape[0] == n_cams and pix_to_face.shape[1] == pix_to_face.shape[2] \
        and pix_to_face.shape[1] % 2 == 0 and pix_to_face.is_contiguous(), "pix_to_face: expected a contiguous (C, 2S, 2S) tensor"
    assert normals.shape == vertices.shape and normals.is_contiguous(), "normals: expected a contiguous (V, 3) tensor"
    S = pix_to_face.shape[1] // 2
    if out is None:
        out = torch.empty(S, n_cams * S, 3, dtype=torch.uint8, device=vertices.device)
    assert out.dim() == 3 and out.shape[0] == S and out.shape[2] == 3 and out.stride(2) == 1 and out.stride(1) == 3 \
        and 0 <= column and (column + n_cams) * S <= out.shape[1], "out: expected an (S, >= (column + C) * S, 3) row-major tensor"
    cells = out[:, column * S:(column + n_cams) * S]
    _launch(_abi.amb_render_shade_normals, 1, _ptr(vertices, torch.float32, "vertices", dev), V,
            _ptr(faces, torch.int32, "faces", dev), F, _ptr(normals, torch.float32, "normals", dev),
            _ptr(cameras, torch.float32, "cameras", dev), n_cams, float(focal), S,
            _ptr(pix_to_face, torch.int32, "pix_to_face", dev), _ptr(cells, torch.uint8, "out", dev), out.stride(0), 3 * S)
    return out


def _icp_tensor(t: torch.Tensor, shape: tuple, name: str) -> None:
    if tuple(t.shape) != shape or not t.is_contiguous():
        raise _lib.AmbError(f"{name}: expected a contiguous {shape} tensor, got {tuple(t.shape)}")


def icp_scratch_doubles(frames: int, candidates: int, n_pred: int, n_gt: int) -> int:
    """Size in fp64 elements of the scratch `icp_chamfer_grad` needs for these sizes."""
    n = C.c_int64()
    _lib.check(_abi.amb_icp_scratch_doubles(int(frames), int(candidates), int(n_pred), int(n_gt), C.byref(n)),
               "amb_icp_scratch_doubles")
    return n.value


def icp_chamfer_grad(pred: torch.Tensor, gt: torch.Tensor, rot: torch.Tensor, params: torch.Tensor,
                     out: Optional[torch.Tensor] = None, scratch: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Chamfer loss and gradient sums of every (frame, candidate) transform -> (F, C, 13) fp64 = loss, t (3), A (3x3).

    pred (F, P, 3), gt (F, Q, 3) fp32; rot (F, C, 3, 3) and params (F, C, 12) = T, d6, s fp32.  The prediction under a
    candidate is (s * x) @ R + T; see include/actionmesh_b200.h for t and A."""
    dev = _device(pred, "pred")
    if pred.dim() != 3 or gt.dim() != 3 or pred.shape[2] != 3 or gt.shape[2] != 3 or gt.shape[0] != pred.shape[0]:
        raise _lib.AmbError(f"icp_chamfer_grad: expected (F, P, 3) and (F, Q, 3) points, got {tuple(pred.shape)} and "
                            f"{tuple(gt.shape)}")
    F, P, Q, nc = pred.shape[0], pred.shape[1], gt.shape[1], params.shape[1] if params.dim() == 3 else 0
    _icp_tensor(pred, (F, P, 3), "pred")
    _icp_tensor(gt, (F, Q, 3), "gt")
    _icp_tensor(rot, (F, nc, 3, 3), "rot")
    _icp_tensor(params, (F, nc, 12), "params")
    need = icp_scratch_doubles(F, nc, P, Q)
    if scratch is None:
        scratch = torch.empty(need, dtype=torch.float64, device=pred.device)
    elif scratch.numel() < need:
        raise _lib.AmbError(f"icp_chamfer_grad: scratch holds {scratch.numel()} doubles, {need} needed")
    if out is None:
        out = torch.empty(F, nc, 13, dtype=torch.float64, device=pred.device)
    _icp_tensor(out, (F, nc, 13), "out")
    _launch(_abi.amb_icp_chamfer_grad, 2, _ptr(pred, torch.float32, "pred", dev), _ptr(gt, torch.float32, "gt", dev), F, nc,
            P, Q, _ptr(rot, torch.float32, "rot", dev), _ptr(params, torch.float32, "params", dev),
            _ptr(scratch, torch.float64, "scratch", dev), _ptr(out, torch.float64, "out", dev),
            tag="icp_chamfer_grad", meta=(F, nc, P, Q))
    return out


def icp_adam_step(sums: torch.Tensor, rot_init: torch.Tensor, step: int, lr: float, params: torch.Tensor,
                  adam_m: torch.Tensor, adam_v: torch.Tensor, rot: torch.Tensor, best: torch.Tensor) -> None:
    """Adam step `step` (1-based) of every (frame, candidate) from `icp_chamfer_grad`'s sums, in place on params, adam_m,
    adam_v (F, C, 12) and rot (F, C, 3, 3), with the best candidate so far tracked in best (F, 16) = loss, R, T, s."""
    dev = _device(sums, "sums")
    if sums.dim() != 3:
        raise _lib.AmbError(f"icp_adam_step: expected (F, C, 13) sums, got {tuple(sums.shape)}")
    F, nc = sums.shape[0], sums.shape[1]
    _icp_tensor(sums, (F, nc, 13), "sums")
    _icp_tensor(rot_init, (nc, 3, 3), "rot_init")
    for t, name in ((params, "params"), (adam_m, "adam_m"), (adam_v, "adam_v")):
        _icp_tensor(t, (F, nc, 12), name)
    _icp_tensor(rot, (F, nc, 3, 3), "rot")
    _icp_tensor(best, (F, 16), "best")
    if step < 1:
        raise _lib.AmbError(f"icp_adam_step: step {step} < 1")
    if rot.data_ptr() == rot_init.data_ptr():
        raise _lib.AmbError("icp_adam_step: rot must not alias rot_init (the step overwrites rot)")
    # torch.optim.Adam computes these scalars in double on the host and applies them to the fp32 state
    step_size = -(float(lr) / (1 - 0.9 ** step))
    bias2_sqrt = (1 - 0.999 ** step) ** 0.5
    _launch(_abi.amb_icp_adam_step, 1, _ptr(sums, torch.float64, "sums", dev), _ptr(rot_init, torch.float32, "rot_init", dev),
            F, nc, step_size, bias2_sqrt, _ptr(params, torch.float32, "params", dev),
            _ptr(adam_m, torch.float32, "adam_m", dev), _ptr(adam_v, torch.float32, "adam_v", dev),
            _ptr(rot, torch.float32, "rot", dev), _ptr(best, torch.float32, "best", dev), tag="icp_adam_step", meta=(F, nc))


def icp_transform_points(points: torch.Tensor, transform: torch.Tensor) -> torch.Tensor:
    """(F, N, 3) fp32 points -> (s * p) @ R + T as pytorch3d's composed Scale / Rotate / Translate applies it, with
    transform (F, 15) or (1, 15) = R (9), T (3), s (3) per frame ((1, 15): the same transform for every frame)."""
    dev = _device(points, "points")
    if points.dim() != 3 or points.shape[2] != 3 or transform.dim() != 2 or transform.shape[1] != 15 \
            or transform.shape[0] not in (1, points.shape[0]) or transform.stride(1) != 1:
        raise _lib.AmbError(f"icp_transform_points: expected (F, N, 3) points and an (F | 1, 15) transform, got "
                            f"{tuple(points.shape)} and {tuple(transform.shape)}")
    p = points.contiguous()
    out = torch.empty_like(p)
    stride = transform.stride(0) if transform.shape[0] > 1 else 0
    _launch(_abi.amb_icp_transform_points, 1 if p.numel() else 0, _ptr(p, torch.float32, "points", dev), p.shape[0],
            p.shape[1], _ptr(transform, torch.float32, "transform", dev), stride, _ptr(out, torch.float32, "out", dev))
    return out


# ---- background removal: RMBG-1.4's resampling, im2col, mask head and refinement (csrc/rmbg.cu) ------------------------------
# Activations are fp32 NHWC feature maps held as 2-D (H * W, pixel stride) tensors with unit channel stride: a GEMM output
# padded to 64 columns is read in place, its first C columns being the channels.
def _feature_map(t: torch.Tensor, h: int, w: int, c: int, name: str) -> None:
    if t.dim() != 2 or t.shape[0] != h * w or t.stride(1) != 1 or t.shape[1] < c or (h * w > 1 and t.stride(0) < c):
        raise _lib.AmbError(f"{name}: expected a ({h * w}, >= {c}) feature map with unit channel stride, got "
                            f"{tuple(t.shape)} strides {t.stride()}")


def _contiguous(t: torch.Tensor, shape: tuple, name: str) -> None:
    if tuple(t.shape) != tuple(shape) or not t.is_contiguous():
        raise _lib.AmbError(f"{name}: expected a contiguous {tuple(shape)} tensor, got {tuple(t.shape)}")


def conv3x3_out(size: int, stride: int, pad: int, dilation: int) -> int:
    return (size + 2 * pad - 2 * dilation - 1) // stride + 1


def rmbg_resize_input(rgb: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """(H, W, 3) uint8 frame -> out (S_h, S_w, 3) fp32 = bilinear(frame) / 255 - 0.5 (background_removal.py:57-69)."""
    dev = _device(rgb, "rgb")
    if rgb.dim() != 3 or rgb.shape[2] != 3:
        raise _lib.AmbError(f"rmbg_resize_input: expected an (H, W, 3) frame, got {tuple(rgb.shape)}")
    _contiguous(rgb, rgb.shape, "rgb")
    if out.dim() != 3:
        raise _lib.AmbError(f"rmbg_resize_input: expected an (S_h, S_w, 3) output, got {tuple(out.shape)}")
    _contiguous(out, (out.shape[0], out.shape[1], 3), "out")
    _launch(_abi.amb_rmbg_resize_input, 1, _ptr(rgb, torch.uint8, "rgb", dev), rgb.shape[0], rgb.shape[1],
            _ptr(out, torch.float32, "out", dev), out.shape[0], out.shape[1], tag="rmbg_resize")
    return out


def rmbg_im2col_split(sources: list, h: int, w: int, out: torch.Tensor, *, stride: int = 1, pad: int = 1,
                      dilation: int = 1) -> torch.Tensor:
    """3x3 patches of the channel concatenation of `sources` = [(feature map, channels)] (one or two) -> out
    (H_o * W_o, 3 k_pad) bf16 in split3's activation layout [hi | lo | hi], k_pad = out.shape[1] / 3."""
    dev = _device(out, "out")
    if not 1 <= len(sources) <= 2:
        raise _lib.AmbError(f"rmbg_im2col_split: one or two sources, got {len(sources)}")
    for i, (t, c) in enumerate(sources):
        _feature_map(t, h, w, c, f"source {i}")
    rows = conv3x3_out(h, stride, pad, dilation) * conv3x3_out(w, stride, pad, dilation)
    if out.dim() != 2 or out.stride(1) != 1 or out.shape[0] != rows or out.shape[1] % 3:
        raise _lib.AmbError(f"rmbg_im2col_split: expected a ({rows}, 3 k_pad) output, got {tuple(out.shape)}")
    (s0, c0), (s1, c1) = sources[0], (sources[1] if len(sources) == 2 else (None, 0))
    _launch(_abi.amb_rmbg_im2col_split, 1, _ptr(s0, torch.float32, "source 0", dev), int(c0), s0.stride(0),
            _ptr(s1, torch.float32, "source 1", dev), int(c1), s1.stride(0) if s1 is not None else 0, h, w, stride, pad,
            dilation, out.shape[1] // 3, _ptr(out, torch.bfloat16, "out", dev), out.stride(0), tag="rmbg_im2col",
            meta=(rows, out.shape[1] // 3))
    return out


def rmbg_maxpool2(src: torch.Tensor, h: int, w: int, c: int, out: torch.Tensor) -> torch.Tensor:
    """MaxPool2d(2, 2, ceil_mode=True) of an (h, w, c) feature map -> out (ceil(h/2) * ceil(w/2), >= c)."""
    dev = _device(src, "src")
    _feature_map(src, h, w, c, "src")
    _feature_map(out, (h + 1) // 2, (w + 1) // 2, c, "out")
    _launch(_abi.amb_rmbg_maxpool2, 1, _ptr(src, torch.float32, "src", dev), src.stride(0), h, w, c,
            _ptr(out, torch.float32, "out", dev), out.stride(0), tag="rmbg_pool")
    return out


def rmbg_upsample(src: torch.Tensor, h: int, w: int, c: int, out: torch.Tensor, out_h: int, out_w: int) -> torch.Tensor:
    """Bilinear (align_corners=False) resize of an (h, w, c) feature map to out (out_h * out_w, >= c)."""
    dev = _device(src, "src")
    _feature_map(src, h, w, c, "src")
    _feature_map(out, out_h, out_w, c, "out")
    _launch(_abi.amb_rmbg_upsample, 1, _ptr(src, torch.float32, "src", dev), src.stride(0), h, w, c,
            _ptr(out, torch.float32, "out", dev), out.stride(0), out_h, out_w, tag="rmbg_upsample")
    return out


def rmbg_mask_head(feat: torch.Tensor, h: int, w: int, weight: torch.Tensor, model_size: tuple, out_size: tuple,
                   work: Optional[dict] = None) -> dict:
    """side1 on the (h, w, 64) stage1d features -> dict(logits (h, w), soft (S_h, S_w) = sigmoid(d1), resized (H, W),
    mask (H, W) uint8) as _postprocess_mask computes it; `work` may hold those tensors (and minmax) to reuse."""
    dev = _device(feat, "feat")
    _feature_map(feat, h, w, 64, "feat")
    _contiguous(weight, (577,), "weight")
    (sh, sw), (oh, ow) = (int(v) for v in model_size), (int(v) for v in out_size)
    work = {} if work is None else work
    for name, shape, dt in (("logits", (h, w), torch.float32), ("soft", (sh, sw), torch.float32),
                            ("resized", (oh, ow), torch.float32), ("mask", (oh, ow), torch.uint8),
                            ("minmax", (2,), torch.int32)):
        if name not in work:
            work[name] = torch.empty(shape, dtype=dt, device=feat.device)
        _contiguous(work[name], shape, name)
    _launch(_abi.amb_rmbg_mask_head, 4, _ptr(feat, torch.float32, "feat", dev), feat.stride(0), h, w,
            _ptr(weight, torch.float32, "weight", dev), _ptr(work["logits"], torch.float32, "logits", dev), sh, sw,
            _ptr(work["soft"], torch.float32, "soft", dev), oh, ow, _ptr(work["resized"], torch.float32, "resized", dev),
            _ptr(work["minmax"], torch.int32, "minmax", dev), _ptr(work["mask"], torch.uint8, "mask", dev),
            tag="rmbg_mask_head")
    return work


def rmbg_refine_rgba(rgb: torch.Tensor, mask: torch.Tensor, refine: bool = True, min_size: int = 200,
                     out: Optional[torch.Tensor] = None, work: Optional[dict] = None) -> torch.Tensor:
    """(H, W, 3) uint8 frame + (H, W) uint8 mask -> (H, W, 4) RGBA with alpha = refine_mask(mask, min_size) (Otsu, 8-connected
    components of >= min_size pixels, 0 / 255) or the mask itself.  `work` receives hist (257: histogram, Otsu threshold),
    labels and sizes (H * W int32 each: component root per foreground pixel, -1 elsewhere; pixels per root)."""
    dev = _device(rgb, "rgb")
    if rgb.dim() != 3 or rgb.shape[2] != 3:
        raise _lib.AmbError(f"rmbg_refine_rgba: expected an (H, W, 3) frame, got {tuple(rgb.shape)}")
    H, W = rgb.shape[0], rgb.shape[1]
    _contiguous(rgb, (H, W, 3), "rgb")
    _contiguous(mask, (H, W), "mask")
    if out is None:
        out = torch.empty(H, W, 4, dtype=torch.uint8, device=rgb.device)
    _contiguous(out, (H, W, 4), "out")
    work = {} if work is None else work
    if refine:
        for name, n in (("hist", 257), ("labels", H * W), ("sizes", H * W)):
            if name not in work:
                work[name] = torch.empty(n, dtype=torch.int32, device=rgb.device)
            _contiguous(work[name], (n,), name)
    get = lambda name: _ptr(work[name], torch.int32, name, dev) if refine else None
    _launch(_abi.amb_rmbg_refine_rgba, 6 if refine else 1, _ptr(rgb, torch.uint8, "rgb", dev),
            _ptr(mask, torch.uint8, "mask", dev), H, W, int(bool(refine)), int(min_size), get("hist"), get("labels"),
            get("sizes"), _ptr(out, torch.uint8, "out", dev), tag="rmbg_refine")
    return out
