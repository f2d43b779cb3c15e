"""Exact-operand restatements of the GEMM (csrc/gemm.cu) and flash-attention (csrc/attention.cu) kernels.

GEMM operands come from dyadic grids: A = i/8 and W = j/16 with |i|, |j| <= 8, so every product is a multiple of 2^-7 with
|p| <= 1/2.  At K <= 8192 every partial sum stays below 2^12 and needs at most 19 significant bits, so the fp32 mainloop is
exact in any accumulation order, and the fp64 matmul of the same operands is the exact accumulator.  The linear epilogue
stays exact too: bias = b/16 and residual = r/8 keep the sums multiples of 2^-7, and col_scale = s/8 (|s| <= 8) gives
multiples of 2^-10 below 2^18.  The kernel's fp32 output must therefore equal the fp64 result bit for bit, and its bf16
output must equal the fp64 result rounded to bf16 (round to nearest even).

GELU, RMSNorm and RoPE cannot be exact.  Their fp64 form is applied to the exact accumulator and each element is held to a
bound derived from the kernel's fp32 operations (u = 2^-24, the unit roundoff of fp32):
  * GELU (gemm.cu gelu_erf): |d| <= 4.2e-7 absolute over |x| <= 12, the error of the Abramowitz-Stegun erfc form with
    fp32 arithmetic (DESIGN 4.2); for |x| > 12 the result is x or a value below 1e-30.
  * RMSNorm: the 128-term fp32 sum of squares has relative error <= 128u, halved by the square root (64u); rsqrtf is
    within 2 ulp (4u); adding eps and the two products rs*w and v*(rs*w) add 2.5u.  So |d| <= 72u * |y|.
  * RoPE: x' = x c - y s and y' = y c + x s round at most three times, each by u (|x| + |y|) since |c|, |s| <= 1, so
    |d| <= 3u (|x| + |y|) for exact x, y; after RMSNorm the inputs carry 72u each: |d| <= 76u (|x| + |y|).
  * A bf16 output adds half a bf16 ulp of |y| + bound.

Canaries: every output, second output, residual, A, W, bias, scale, norm weight and rope table is a view into a wider
buffer whose hidden elements hold a NaN bit pattern.  A read past k, n or the rope table reaches a NaN and shows up in the
result; a write outside the rows a call owns (rows >= m, the gaps of a row map, the padding columns) changes a NaN.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Optional

import torch

U = 2.0 ** -24
GELU_ABS = 4.2e-7
NORM_REL = 72 * U
ROPE_REL = 3 * U
ROPE_NORMED_REL = 76 * U
NORM_EPS = 1e-6

NAN_BF16 = 0x7FCA       # quiet NaN with a payload no arithmetic produces
NAN_F32 = 0x7FCAFE01
PAD_COLS = 64           # hidden columns of every padded view (one 128-byte TMA box row of bf16)
PAD_ROWS = 3            # spare rows below every padded output

# row maps (grp_rows, grp_stride, row_off) as the pipeline launches them: proj_in rows (frame, token) -> h rows (frame,
# 1 + token) (denoiser.py), the time token (1, L, 0), DinoV2's patch rows behind the class token (image_encoder.py) and
# Stage II's post_quant rows in front of the alpha token (autoencoder.py)
ROW_MAPS = {"tokens": (31, 32, 1), "time": (1, 5, 0), "patch": (16, 17, 1), "frames": (31, 32, 0)}

# M values of every configuration: one row, the tile edges, an odd count of 128-row tiles (the last cluster pair has an
# empty peer), and 161 ragged tiles: 81 pairs over 11 raster bands of 8 pairs, more units than clusters, so every
# consumer warpgroup runs several tiles
SMALL_MS = (1, 127, 128, 129, 640, 161 * 128 - 45)


def int_view(t: torch.Tensor) -> torch.Tensor:
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def nan_bits(dtype) -> int:
    return NAN_BF16 if dtype == torch.bfloat16 else NAN_F32


def nan_buffer(shape, dtype, device) -> torch.Tensor:
    t = torch.empty(shape, dtype=dtype, device=device)
    int_view(t).fill_(nan_bits(dtype))
    return t


def is_untouched(buf: torch.Tensor) -> bool:
    return bool((int_view(buf) == nan_bits(buf.dtype)).all())


def grid(shape, imax: int, den: int, gen: torch.Generator, device, dtype=torch.bfloat16) -> torch.Tensor:
    """Integers in [-imax, imax] divided by the power of two `den`: exactly representable in bf16 and fp32."""
    i = torch.randint(-imax, imax + 1, shape, generator=gen, device=device, dtype=torch.int32)
    return i.to(dtype) / den


def padded(values: torch.Tensor, pad_cols: int = PAD_COLS, pad_rows: int = 0) -> tuple[torch.Tensor, torch.Tensor]:
    """(buffer, view): `values` in the top-left corner of a NaN-filled buffer with extra columns and rows."""
    r, c = values.shape
    buf = nan_buffer((r + pad_rows, c + pad_cols), values.dtype, values.device)
    buf[:r, :c] = values
    return buf, buf[:r, :c]


def padded_vector(values: torch.Tensor, pad: int = PAD_COLS) -> torch.Tensor:
    buf = nan_buffer((values.numel() + pad,), values.dtype, values.device)
    buf[:values.numel()] = values
    return buf[:values.numel()]


def half_ulp_bf16(y: torch.Tensor) -> torch.Tensor:
    """Half a bf16 ulp at |y| (8 significant bits): 2^(e - 9) for |y| in [2^(e-1), 2^e)."""
    _, e = torch.frexp(y.abs())
    return torch.where(y == 0, torch.zeros_like(y), torch.ldexp(torch.ones_like(y), e - 9))


def gelu64(x: torch.Tensor) -> torch.Tensor:
    return 0.5 * x * torch.erfc(-x / math.sqrt(2.0))


def compare(got: torch.Tensor, exp: torch.Tensor, bound: Optional[torch.Tensor], what: str, store_rounding: bool = True) -> None:
    """Exact: the output's bits equal those of the fp64 value in the output's type (and, for fp32, the fp64 value is an
    fp32 number: the exactness premise).  Bounded: |got - exp| <= bound element by element."""
    if bound is None:
        if got.dtype == torch.float32:
            assert torch.equal(exp.float().double(), exp), f"{what}: the exact result is not an fp32 number (grid premise)"
        want = exp.to(got.dtype)
        eq = int_view(got) == int_view(want)
        if not bool(eq.all()):
            i = (~eq).nonzero()[0].tolist()
            raise AssertionError(f"{what}: {int((~eq).sum())} elements differ from the exact result, first at {i}: "
                                 f"got {got[tuple(i)].item()!r}, want {want[tuple(i)].item()!r}")
        return
    if got.dtype == torch.bfloat16 and store_rounding:
        bound = bound + half_ulp_bf16(exp.abs() + bound)
    err = (got.double() - exp).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        i = bad.nonzero()[0].tolist()
        t = tuple(i)
        raise AssertionError(f"{what}: {int(bad.sum())} elements outside the bound, first at {i}: got {got[t].item()!r}, "
                             f"want {exp[t].item()!r}, |d| = {err[t].item():.3e} > {bound[t].item():.3e}")


# ---------------------------------------------------------------------------------------------------------------- GEMM
@dataclass(frozen=True)
class GemmConfig:
    """One epilogue configuration of ops.gemm.  residual: None, "alias" (the output itself) or "other" (another buffer);
    norm: None, "q" (all columns one weight), "q_rope" (the same + RoPE), "kv" (first half normed), "kv_rope" (first half normed + RoPE), "qkv"
    (two thirds, two weights), "qkv_rope" (the same + RoPE), "rope" (RoPE on two thirds, no norm)."""
    name: str
    n: int
    k: int
    out: str = "bf16"
    bias: bool = False
    act: int = 0
    col_scale: bool = False
    residual: Optional[str] = None
    res: str = "bf16"
    out2: bool = False
    row_map: Optional[str] = None
    k_split: Optional[int] = None
    norm: Optional[str] = None
    rows_per_pos: int = 33


GEMM_CONFIGS = [
    GemmConfig("plain_bf16", 256, 128),
    GemmConfig("plain_f32", 256, 128, out="f32"),
    GemmConfig("bias_bf16", 256, 128, bias=True),
    GemmConfig("bias_f32", 256, 128, out="f32", bias=True),
    GemmConfig("bias_gelu_bf16", 512, 128, bias=True, act=1),
    GemmConfig("bias_gelu_f32", 512, 128, out="f32", bias=True, act=1),
    # DinoV2 LayerScale blocks: x = x + ls * (a W^T + b), in place
    GemmConfig("ls_res_alias_bf16", 256, 128, bias=True, col_scale=True, residual="alias"),
    GemmConfig("ls_res_alias_f32", 256, 128, out="f32", bias=True, col_scale=True, residual="alias", res="f32"),
    # the residual stream in place: bf16, fp32, and fp32 with its bf16 operand copy (denoiser ff2)
    GemmConfig("bias_res_alias_bf16", 256, 128, bias=True, residual="alias"),
    GemmConfig("bias_res_alias_f32", 256, 128, out="f32", bias=True, residual="alias", res="f32"),
    GemmConfig("bias_res_alias_f32_out2", 256, 128, out="f32", bias=True, residual="alias", res="f32", out2=True),
    # residual from another buffer: residual=h_in (denoiser), residual=qp (Stage II)
    GemmConfig("bias_res_other_bf16", 256, 128, bias=True, residual="other"),
    GemmConfig("bias_res_other_f32", 256, 128, out="f32", bias=True, residual="other", res="f32"),
    GemmConfig("bias_res_other_bf16_to_f32", 256, 128, out="f32", bias=True, residual="other"),
    # row maps
    GemmConfig("rowmap_tokens_bf16", 256, 128, bias=True, row_map="tokens"),
    GemmConfig("rowmap_tokens_f32", 256, 128, out="f32", bias=True, row_map="tokens"),
    GemmConfig("rowmap_time_bf16", 256, 128, bias=True, row_map="time"),
    GemmConfig("rowmap_time_f32", 256, 128, out="f32", bias=True, row_map="time"),
    GemmConfig("rowmap_patch_res_bf16", 256, 128, bias=True, residual="alias", row_map="patch"),
    GemmConfig("rowmap_patch_res_f32", 256, 128, out="f32", bias=True, residual="alias", res="f32", row_map="patch"),
    GemmConfig("rowmap_frames_bf16", 256, 128, bias=True, row_map="frames"),
    GemmConfig("rowmap_frames_f32", 256, 128, out="f32", bias=True, row_map="frames"),
    # two A sources (denoiser skip linear): the split at the first k-block, the middle, the last k-block
    GemmConfig("a2_split64_bf16", 256, 256, bias=True, k_split=64),
    GemmConfig("a2_split_half_bf16", 256, 256, bias=True, k_split=128),
    GemmConfig("a2_split_last_bf16", 256, 256, bias=True, k_split=192),
    GemmConfig("a2_split_half_f32", 256, 256, out="f32", bias=True, k_split=128),
    # per-head epilogues
    GemmConfig("q_norm", 256, 128, norm="q"),
    GemmConfig("q_norm_rope", 256, 128, norm="q_rope"),
    GemmConfig("kv_norm", 512, 128, norm="kv"),
    GemmConfig("kv_norm_rope", 512, 128, norm="kv_rope"),
    GemmConfig("qkv_norm", 768, 128, norm="qkv"),
    GemmConfig("qkv_norm_rope", 768, 128, norm="qkv_rope"),
    GemmConfig("rope_only", 768, 128, norm="rope"),
    GemmConfig("rope_only_one_row_per_pos", 384, 128, norm="rope", rows_per_pos=1),
    # BN = 64 (n not a multiple of 128) with more than one N tile, and a single one
    GemmConfig("bn64_n64_bias_f32", 64, 128, out="f32", bias=True),
    GemmConfig("bn64_n64_bias_bf16", 64, 128, bias=True),
    GemmConfig("bn64_n192_res_f32", 192, 128, out="f32", bias=True, residual="alias", res="f32"),
    GemmConfig("bn64_n320_res_f32", 320, 128, out="f32", bias=True, residual="alias", res="f32"),
    GemmConfig("bn64_n320_res_bf16", 320, 128, bias=True, residual="alias"),
    # Stage II's score GEMM S = Q'K'^T and V-transpose GEMM V^T = W_v ctx^T: fp32, no bias, N = Rp = 64 mod 128
    GemmConfig("bn64_n192_f32", 192, 128, out="f32"),
]
GEMM_CONFIG = {c.name: c for c in GEMM_CONFIGS}


def _norm_layout(cfg: GemmConfig) -> tuple[int, int, int]:
    """(norm_cols, norm_seg, rope_cols) of a per-head configuration."""
    n = cfg.n
    return {"q": (n, n, 0), "q_rope": (n, n, n), "kv": (n // 2, n // 2, 0), "kv_rope": (n // 2, n // 2, n // 2), "qkv": (2 * n // 3, n // 3, 0),
            "qkv_rope": (2 * n // 3, n // 3, 2 * n // 3), "rope": (0, 0, 2 * n // 3)}[cfg.norm]


def row_map_rows(cfg: GemmConfig, m: int) -> tuple[Optional[tuple[int, int, int]], int]:
    """(row_map or None, output rows the call needs)."""
    if cfg.row_map is None:
        return None, m
    g, s, o = ROW_MAPS[cfg.row_map]
    return (g, s, o), ((m - 1) // g) * s + (m - 1) % g + o + 1


def dest_rows(row_map, m: int, device) -> torch.Tensor:
    r = torch.arange(m, device=device)
    if row_map is None:
        return r
    g, s, o = row_map
    return (r // g) * s + r % g + o


@dataclass
class GemmCase:
    cfg: GemmConfig
    m: int
    a: torch.Tensor
    w: torch.Tensor
    out: torch.Tensor
    out_buf: torch.Tensor
    kw: dict = field(default_factory=dict)
    out2_buf: Optional[torch.Tensor] = None
    res_values: Optional[torch.Tensor] = None  # the residual rows drow as they were before the call
    drow: Optional[torch.Tensor] = None

    def call(self, gemm) -> None:
        gemm(self.a, self.w, self.out, **self.kw)


def build_gemm_case(cfg: GemmConfig, m: int, device, seed: int = 0, pad: bool = True) -> GemmCase:
    """Operands of one call on the exact grids.  pad=False gives contiguous, exactly sized tensors (ldc == n); the output
    still has spare rows."""
    gen = torch.Generator(device=device).manual_seed(seed)
    n, k = cfg.n, cfg.k
    pc = PAD_COLS if pad else 0
    dt = {"bf16": torch.bfloat16, "f32": torch.float32}
    a_full = grid((m, k), 8, 8, gen, device)
    w = grid((n, k), 8, 16, gen, device)
    kw = {}
    if cfg.k_split is not None:
        _, a = padded(a_full[:, :cfg.k_split].contiguous(), pc, PAD_ROWS if pad else 0)
        _, kw["a2"] = padded(a_full[:, cfg.k_split:].contiguous(), pc, PAD_ROWS if pad else 0)
    else:
        _, a = padded(a_full, pc, PAD_ROWS if pad else 0)
    _, w = padded(w, pc)
    if cfg.bias:
        kw["bias"] = padded_vector(grid((n,), 8, 16, gen, device, torch.float32), pc)
    if cfg.act:
        kw["act"] = cfg.act
    if cfg.col_scale:
        kw["col_scale"] = padded_vector(grid((n,), 8, 8, gen, device, torch.float32), pc)
    row_map, rows = row_map_rows(cfg, m)
    if row_map is not None:
        kw["row_map"] = row_map
    out_buf = nan_buffer((rows + PAD_ROWS, n + pc), dt[cfg.out], device)
    out = out_buf[:rows, :n]
    drow = dest_rows(row_map, m, device)
    res_values = None
    if cfg.residual is not None:
        rv = grid((rows, n), 8, 8, gen, device, dt[cfg.res])
        if cfg.residual == "alias":
            assert cfg.res == cfg.out
            out_buf[drow, :n] = rv[drow]
            kw["residual"] = out
        else:
            _, kw["residual"] = padded(rv, pc, PAD_ROWS)
        res_values = rv[drow]
    out2_buf = None
    if cfg.out2:
        out2_buf = nan_buffer((rows + PAD_ROWS, n + pc + 8), torch.bfloat16, device)  # its own row stride
        kw["out2"] = out2_buf[:rows, :n]
    if cfg.norm is not None:
        nc, seg, rc = _norm_layout(cfg)
        d = dict(cols=nc, seg=seg, eps=NORM_EPS, rope_cols=rc, rows_per_pos=cfg.rows_per_pos)
        if nc:
            d["w0"] = padded_vector(grid((128,), 8, 8, gen, device, torch.float32) + 2.0, pc)
            if seg < nc:
                d["w1"] = padded_vector(grid((128,), 8, 8, gen, device, torch.float32) - 2.0, pc)
        if rc:
            npos = (m + cfg.rows_per_pos - 1) // cfg.rows_per_pos
            ang = torch.rand(npos, 64, generator=gen, device=device) * 6.2832
            _, d["cos"] = padded(ang.cos(), 0, PAD_ROWS)
            _, d["sin"] = padded(ang.sin(), 0, PAD_ROWS)
        kw["norm"] = d
    return GemmCase(cfg, m, a, w, out, out_buf, kw, out2_buf, res_values, drow)


def gemm_expected(case: GemmCase, r0: int, r1: int) -> list[tuple[slice, torch.Tensor, Optional[torch.Tensor]]]:
    """fp64 results of rows [r0, r1) as (column slice, value, bound or None for exact)."""
    cfg, kw = case.cfg, case.kw
    a = case.a[r0:r1].double()
    if "a2" in kw:
        a = torch.cat([a, kw["a2"][r0:r1].double()], 1)
    acc = a @ case.w.double().t()
    parts = []
    c_lin = 0
    if cfg.norm is not None:
        nc, seg, rc = _norm_layout(cfg)
        d = kw["norm"]
        pos = torch.arange(r0, r1, device=acc.device) // cfg.rows_per_pos
        for c0 in range(0, max(nc, rc), 128):
            x = acc[:, c0:c0 + 128]
            bound = torch.zeros_like(x)
            if c0 < nc:
                wn = (d["w0"] if c0 < seg else d.get("w1", d["w0"])).double()
                ms = x.pow(2).mean(-1, keepdim=True) + float(torch.tensor(NORM_EPS, dtype=torch.float32))
                x = x / ms.sqrt() * wn
                bound = NORM_REL * x.abs()
            if c0 < rc:
                cs, sn = d["cos"][pos].double(), d["sin"][pos].double()
                x0, x1 = x[:, 0::2], x[:, 1::2]
                mag = x0.abs() + x1.abs()
                rel = ROPE_NORMED_REL if c0 < nc else ROPE_REL
                x = torch.stack([x0 * cs - x1 * sn, x1 * cs + x0 * sn], -1).flatten(1)
                bound = (rel * mag).repeat_interleave(2, dim=1)
            parts.append((slice(c0, c0 + 128), x, bound))
        c_lin = max(nc, rc)
    if c_lin < cfg.n:
        v = acc[:, c_lin:]
        if "bias" in kw:
            v = v + kw["bias"][c_lin:].double()
        bound = None
        if cfg.act:
            v = gelu64(v)
            bound = torch.full_like(v, GELU_ABS)
        if "col_scale" in kw:
            v = v * kw["col_scale"][c_lin:].double()
        if case.res_values is not None:
            v = v + case.res_values[r0:r1, c_lin:].double()
        parts.append((slice(c_lin, cfg.n), v, bound))
    return parts


def check_gemm(case: GemmCase, chunk_elems: int = 1 << 26) -> None:
    """Every element of the output (and out2) against gemm_expected, in row chunks; then every element the call does not
    own must still hold its NaN bit pattern.  Overwrites the checked rows with NaN as it goes."""
    cfg = case.cfg
    step = max(1, chunk_elems // max(cfg.n, cfg.k))
    for r0 in range(0, case.m, step):
        r1 = min(case.m, r0 + step)
        rows = case.drow[r0:r1]
        got = case.out_buf[rows, :cfg.n]
        got2 = case.out2_buf[rows, :cfg.n] if case.out2_buf is not None else None
        for cols, exp, bound in gemm_expected(case, r0, r1):
            what = f"{cfg.name} m={case.m} rows [{r0}, {r1}) cols [{cols.start}, {cols.stop})"
            compare(got[:, cols], exp, bound, what)
            if got2 is not None:
                compare(got2[:, cols], exp, bound, what + " out2")
        int_view(case.out_buf)[rows, :cfg.n] = nan_bits(case.out_buf.dtype)
        if case.out2_buf is not None:
            int_view(case.out2_buf)[rows, :cfg.n] = NAN_BF16
    assert is_untouched(case.out_buf), f"{cfg.name} m={case.m}: wrote outside its rows / columns"
    if case.out2_buf is not None:
        assert is_untouched(case.out2_buf), f"{cfg.name} m={case.m}: out2 written outside its rows / columns"


def gemm_signature(a, w, out, *, bias=None, a2=None, residual=None, act=0, col_scale=None, row_map=None, norm=None,
                   out2=None, tag=None) -> tuple:
    """The epilogue configuration of one ops.gemm call, free of sizes: what a kernel-level test has to have exercised."""
    n = w.shape[0]
    if residual is None:
        res = None
    else:
        alias = residual.data_ptr() == out.data_ptr() and residual.stride() == out.stride()
        res = ("alias" if alias else "other", str(residual.dtype).split(".")[-1])
    rm = None if row_map is None else ("grp1" if row_map[0] == 1 else "grpN", "off%d" % row_map[2])
    nrm = None
    if norm is not None:
        nc, rc = norm.get("cols", 0), norm.get("rope_cols", 0)
        frac = lambda c: "none" if c == 0 else ("all" if c == n else "part")
        nrm = (frac(nc), norm.get("w1") is not None, frac(rc))
    return (("out", str(out.dtype).split(".")[-1]), ("bias", bias is not None), ("act", act), ("col_scale", col_scale is not None),
            ("residual", res), ("out2", out2 is not None), ("row_map", rm), ("norm", nrm), ("a2", a2 is not None),
            ("strided", out.stride(0) != n), ("bn", 128 if n % 128 == 0 else 64))


def table_signatures(device="cpu") -> set:
    """Signatures of every GEMM_CONFIGS row, padded and contiguous (the two layouts the exactness tests run)."""
    sigs = set()
    for cfg in GEMM_CONFIGS:
        for pad in (True, False):
            c = build_gemm_case(cfg, 129, device, pad=pad)
            sigs.add(gemm_signature(c.a, c.w, c.out, **c.kw))
    return sigs


# ---------------------------------------------------------------------------------------------------------- attention
def attn_tensor(B, S, H, D, gen, device, *, chunks=1, kind="normal", scale=1.0) -> torch.Tensor:
    """(B, S, H, D) or (B, chunks, S / chunks, H, D) bf16 view into a buffer with PAD_COLS NaN columns after every head and
    PAD_ROWS NaN rows after every sequence.  kind "normal": N(0, scale²); "uniform": U[0.5, 1.5)."""
    shape = (B, S, H, D) if chunks == 1 else (B, chunks, S // chunks, H, D)
    vals = torch.randn(shape, generator=gen, device=device) * scale if kind == "normal" else \
        torch.rand(shape, generator=gen, device=device) + 0.5
    bshape = list(shape)
    bshape[-3] += PAD_ROWS
    bshape[-1] += PAD_COLS
    buf = nan_buffer(tuple(bshape), torch.bfloat16, device)
    view = buf[..., :shape[-3], :, :D]
    view.copy_(vals)
    return view


def attn_out(B, Sq, H, D, device) -> tuple[torch.Tensor, torch.Tensor]:
    buf = nan_buffer((B, Sq + PAD_ROWS, H, D + PAD_COLS), torch.bfloat16, device)
    return buf, buf[:, :Sq, :, :D]


def sample_rows(Sq: int, gen: torch.Generator, n_random: int = 64) -> torch.Tensor:
    """Every row of the last 128-row query tile, the rows on both sides of every 128-row boundary, random rows."""
    last0 = (Sq - 1) // 128 * 128
    rows = set(range(last0, Sq))
    for b in range(128, Sq, 128):
        rows.update((b - 1, b))
    rows.update(torch.randint(0, Sq, (n_random,), generator=gen).tolist())
    return torch.tensor(sorted(rows))


def attn_bound_rows(q, k, v, scale, b, h, rows, tiles):
    """(o64 (R, D), bound (R, D)) for query rows `rows` of (batch b, head h); k, v as (Sk, D) of that (b, h).

    The kernel divides sum_k bf16(p_k) v_k by l = sum_k p_k with p_k = exp2(fp32 logit terms) and stores bf16:
      * rounding P to bf16 moves each p_k by <= 2^-9 p_k: <= 2^-9 max_k |v_kd| on the output;
      * the bf16 store: <= 2^-9 |o|;
      * every p_k carries a relative error e: the fp32 S = q.k (D exact products, accumulated with <= 2u per add)
        moves the logit by scale * 2 D u sum_d |q_d k_d|; the fp32 exponent argument s c - m c by 3u sigma (sigma =
        max_k |scale S_k|); ex2.approx by 2^-22.  Errors shared by numerator and denominator cancel to first order, so
        the output moves by <= 2 e max_k |v_kd|;
      * fp32 accumulation: o over 128 keys per tile and the running rescales, l over 32 terms per thread and tile:
        (2 * 128 + 4 * tiles + 40) u of max_k |v_kd|.
    """
    qs = q[b, rows, h].double()
    kk, vv = k.double(), v.double()
    s = qs @ kk.t() * scale
    o64 = torch.softmax(s, -1) @ vv
    sigma = s.abs().amax(-1, keepdim=True)
    qk_abs = (qs.abs() @ kk.abs().t()).amax(-1, keepdim=True) * scale
    D = q.shape[-1]
    e = 2 * D * U * qk_abs + 3 * U * sigma + 2.0 ** -22
    vmax = vv.abs().amax(0, keepdim=True)
    bound = (2.0 ** -9 + 2 * e + (2 * 128 + 4 * tiles + 40) * U) * vmax + 2.0 ** -9 * o64.abs()
    return o64, bound
