"""Restatements and per-element error bounds of the fp32-grade split-bf16 path: csrc/elementwise.cu split3_kernel and
softmax_split3_kernel, the GEMM (csrc/gemm.cu) on split operands, and csrc/attention_small.cu.  u = 2^-24 throughout.

split3.  hi = RN_bf16(x) and lo = RN_bf16(x - hi); x - hi is exact in fp32.  For x in [2^e, 2^(e+1)), |x - hi| <= 2^(e-8)
(half a bf16 ulp), so |lo| <= 2^(e-8) and |x - hi - lo| <= half a bf16 ulp of a number below 2^(e-8): <= 2^(e-17) <=
2^-17 |x| (a remainder of exactly 2^(e-8) is a power of two and splits without error).  Below 2^-126 the bf16 spacing is
2^-133, so the split is only good to 2^-134 absolute: SPLIT_REL |x| + SPLIT_ABS.  The A operand is [hi | lo | hi], the W
operand [hi | hi | lo], per segment of `seg` columns, so A' W'^T = sum a_hi w_hi + a_lo w_hi + a_hi w_lo.

Exact split grid.  hi = i/8 with i in {0, +-5, +-6, +-7} and lo = j/2^L with |j| <= 2^(L-9) - 1 (lo = 0 where hi = 0).
hi lies in [5/8, 7/8], where half a bf16 ulp is 2^-9 > |lo|, and x = hi + lo has at most L bits below the point, so
split3 returns exactly (hi, lo).  Every product is a multiple of 2^-(L+3) (hi hi = i i'/64, hi lo = i j / 2^(L+3)); one
logical term a_hi w_hi + a_lo w_hi + a_hi w_lo is below 49/64 + 2 (7/8) 2^-9 < 0.769 in magnitude, so every partial sum
of any subset of the 3K products, in any order, is below 0.769 K and needs b + L + 3 bits with 2^b > 0.769 K.  L = 12
keeps that within fp32's 24 bits up to K = 512 (b = 9; K = 128, the score GEMM's 3 x 128 columns, needs 22), L = 11 up to
K = 1024 (b = 10, 24 bits).  The kernel's fp32 accumulation is then exact, and the fp64 value of
sum(a_hi w_hi + a_lo w_hi + a_hi w_lo) (the exact product minus the dropped a_lo w_lo) is the result bit for bit.

Split GEMM at long K.  Against the fp64 product of the unsplit fp32 operands, per output element:
  * representation: a w - (a_hi w_hi + a_lo w_hi + a_hi w_lo) = a_lo w_lo + (a_hi + a_lo) dw + da (w_hi + w_lo) + da dw
    with |a_lo| <= 2^-8 |a|, |da| <= 2^-17 |a| (likewise w): <= 2^-16 + 2 (2^-17 + 2^-34) + 2^-34 < 2^-15 (1 + 2^-15) of
    |a||w| per term: SPLIT_GEMM_REP sum |a||w|;
  * accumulation: one fp32 accumulator per element takes the K' = 3K columns in order, 16 per wgmma step (s = K'/16
    steps).  The Hopper tensor core adds the 16 exact products to the accumulator and rounds the result once, toward zero
    in the worst case: <= 2u (|S_(j-1)| + sum of the step's |products|), S_j the partial sums.  A logical term k has its
    three products in steps >= k // 16 (its hi hi product is in column k of a one-segment operand), so
    sum_j |S_j| <= sum_k (s - k // 16) |a_k w_k| (1 + 2^-7): WGMMA_STEP * sum_k (s - k // 16) |a_k||w_k|.  The weight is
    what keeps the bound tight: the last two thirds of the steps add only lo products to a nearly complete sum, and the
    weighted sum is 5/6 of s sum |a||w| instead of s sum |a||w|.
  At K' = 98 496 (P'V'^T of Stage II's default window, s = 6156) the bound is at most (2^-15 + 2u 6156 (1 + 2^-7))
  sum |a||w| = 7.6e-4 sum |a||w|, and 6.4e-4 sum |a||w| for same-sign operands, where it is attained in shape.  A missing
  hi-lo cross term costs sum a_lo w_hi, up to 2^-9 sum |a||w| = 1.95e-3 sum |a||w| when the lo parts share the products'
  sign: 2.6 to 3 times the bound.
  The fused epilogue adds one rounding per step (bias, GELU, column scale, residual): epilogue_bound.

softmax_split3.  Row r, y_k = x_k scale (exact in fp64), Y = max |y_k|, sigma = max y - min y over the n live columns,
G = ceil(n / 2048) float4 groups per thread.  The kernel's p = expf(fl(y) - M) / L with M = fl(max y):
  * the exponent argument carries u |y_k| + u |M| + u |y_k - M| <= u (2Y + sigma) (a fused multiply-add only removes a
    rounding); expf is within 2 ulp (4u) without fast-math;
  * L: every term's exponent (2uY for fl(y_k) and M, and the telescoping rescale arguments m_old - m_new: u sigma at the
    thread, warp and CTA level, 3u sigma), G + 7 expf calls (4u each), G + 6 rescale products and G + 24 additions of
    positive terms on any term's path (3 within a float4, G into the thread's l, 5 across the warp, 16 across the CTA):
    u (2Y + 4 sigma + 6G + 58);
  * 1/L and the product with it: 2u.
  So p = p64 (1 + e), |e| <= u (4Y + 5 sigma + 6G + 64) (x 1.01 for second-order terms), and p_hi + p_lo adds SPLIT_REL.
  Below 2^-126 expf loses its relative accuracy: SOFTMAX_ABS = 2^-133 absolute covers expf, the product and the split.

attn_small_f32.  Per (frame, head), s_k = q . k_k in fp32 (64 fmaf in order: |ds_k| <= 65u sum_d |q_d k_kd|), m = max s~
(a common shift, whose own error cancels in the softmax), p~_k = expf(fl(fl(s~_k - m) scale)): the logit moves by
d_k <= scale (65u sum_d |q_d k_kd| + 2.01u (max s - s_k)), and p~_k = P_k (1 + eps_k), |eps_k| <= 1.01 d_k + 4.01u.
With pi = softmax, o~ - o = sum_k P_k eps_k (v_k - o) / sum_k P~_k exactly, so |o~ - o| <= sum_k pi_k |eps_k| (|v_k| + |o|)
(1.01).  The output accumulates S products by fmaf in key order (<= S u sum pi |v|), the row sum adds <= 10 terms per lane
and 5 butterfly steps (15u), 1/sum and the last product 2u: + S u (pi @ |V|) + 17u |o|.

How tight the bounds are (largest |error| / bound on an H100, at the shapes of tests/test_fp32_grade_gpu.py): softmax_split3
0.49 to 0.63 (the split's 2^-17 dominates); P'V'^T at K' = 98 496 with one-sign operands 0.56; the score GEMM (K' = 384)
0.13; attn_small_f32 0.010 to 0.026 and the split GEMMs on mixed-sign operands at K' = 3072 and 12 288 (V-transpose,
Stage II ff2, DinoV2-L qkv / ff1 / ff2) 0.033 to 0.046.  The last two are worst cases of
n roundings of one sign (the 64-term dot products, the S-term output sum, the K'/16 accumulation steps), which grow like n;
the rounding errors of mixed-sign or random data grow like sqrt(n), and P'V'^T shows the same bound met within 2x when
the signs do line up.
"""
from __future__ import annotations

import math

import torch

import kernel_exact as kx

U = kx.U
SPLIT_REL = 2.0 ** -17
SPLIT_ABS = 2.0 ** -134
SPLIT_GEMM_REP = 2.0 ** -15 * (1 + 2.0 ** -15)
WGMMA_STEP = 2 * U * (1 + 2.0 ** -7)
SOFTMAX_ABS = 2.0 ** -133
GRID_TERM_MAX = 0.769


# ------------------------------------------------------------------------------------------------------------- split3
def split_parts(x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """(hi, lo) bf16 of fp32 x, with torch's round-to-nearest-even conversion."""
    hi = x.to(torch.bfloat16)
    return hi, (x - hi.float()).to(torch.bfloat16)


def split_layout(x: torch.Tensor, seg: int | None = None, weight: bool = False) -> torch.Tensor:
    """The (rows, 3 cols) bf16 operand split3 writes: each segment of `seg` columns becomes [hi|lo|hi] (activation) or
    [hi|hi|lo] (weight)."""
    rows, cols = x.shape
    seg = seg or cols
    hi, lo = split_parts(x)
    parts = (hi, hi, lo) if weight else (hi, lo, hi)
    return torch.stack([p.view(rows, cols // seg, seg) for p in parts], 2).reshape(rows, 3 * cols)


def lo_bits(k: int) -> int:
    """L of the exact split grid for a logical depth K (module docstring)."""
    b = math.ceil(math.log2(GRID_TERM_MAX * k))
    L = min(12, 21 - b)
    assert L >= 10, f"K = {k} is too deep for the exact split grid"
    return L


def split_grid(shape, k: int, gen: torch.Generator, device) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """(x fp32, hi fp32, lo fp32) on the exact split grid for depth k."""
    L = lo_bits(k)
    jmax = 2 ** (L - 9) - 1
    vals = torch.tensor([0.0, 5, 6, 7, -5, -6, -7], device=device)
    hi = vals[torch.randint(0, 7, shape, generator=gen, device=device)] / 8
    lo = torch.randint(-jmax, jmax + 1, shape, generator=gen, device=device).float() / 2 ** L
    lo = torch.where(hi == 0, torch.zeros_like(lo), lo)
    return hi + lo, hi, lo


# ---------------------------------------------------------------------------------------------------------- split GEMM
def split_gemm_bound(a: torch.Tensor, w: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """(c64, bound) of A' W'^T for fp32-valued rows a (m, K) and w (n, K), one segment each (module docstring)."""
    a64, w64 = a.double(), w.double()
    K = a.shape[1]
    s = 3 * K // 16
    weight = (s - torch.arange(K, device=a.device) // 16).double()
    aa, wa = a64.abs(), w64.abs().t()
    return a64 @ w64.t(), SPLIT_GEMM_REP * (aa @ wa) + WGMMA_STEP * ((aa * weight) @ wa)


def epilogue_bound(acc: torch.Tensor, acc_bound: torch.Tensor, bias=None, act: int = 0, col_scale=None, residual=None):
    """(value, bound) of the fused epilogue bias -> GELU -> column scale -> + residual applied to an fp64 accumulator
    known to within acc_bound; one fp32 rounding per step (kernel_exact.GELU_ABS for the erfc form, slope <= 1.13)."""
    v, b = acc, acc_bound
    if bias is not None:
        v = v + bias.double()
        b = b + U * v.abs()
    if act:
        v = kx.gelu64(v)
        b = 1.13 * b + kx.GELU_ABS + U * v.abs()
    if col_scale is not None:
        s = col_scale.double()
        v = v * s
        b = b * s.abs() + U * v.abs()
    if residual is not None:
        v = v + residual.double()
        b = b + U * v.abs()
    return v, b


# ---------------------------------------------------------------------------------------------------- softmax_split3
def softmax_bound(x: torch.Tensor, scale: float) -> tuple[torch.Tensor, torch.Tensor]:
    """(p64, bound on |p_hi + p_lo - p64|) of the rows of fp32 scores x (rows, n) (module docstring)."""
    y = x.double() * float(torch.tensor(scale, dtype=torch.float32))
    n = x.shape[1]
    Y = y.abs().amax(-1, keepdim=True)
    sigma = y.amax(-1, keepdim=True) - y.amin(-1, keepdim=True)
    G = (n + 2047) // 2048
    e = 1.01 * U * (4 * Y + 5 * sigma + 6 * G + 64)
    p = torch.softmax(y, -1)
    return p, p * (e + SPLIT_REL * (1 + e)) + SOFTMAX_ABS


# ----------------------------------------------------------------------------------------------------- attn_small_f32
def attn_small_bound(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, scale: float) -> tuple[torch.Tensor, torch.Tensor]:
    """(o64, bound) of softmax(scale q k^T) v for (B, S, 64) fp32 q, k, v (module docstring)."""
    q64, k64, v64 = q.double(), k.double(), v.double()
    S = q.shape[-2]
    sc = float(torch.tensor(scale, dtype=torch.float32))
    s = q64 @ k64.transpose(-1, -2)
    pi = torch.softmax(s * sc, -1)
    o = pi @ v64
    d = sc * (65 * U * (q64.abs() @ k64.abs().transpose(-1, -2)) + 2.01 * U * (s.amax(-1, keepdim=True) - s))
    pe = pi * (1.01 * d + 4.01 * U)
    va = v64.abs()
    bound = 1.01 * (pe @ va + pe.sum(-1, keepdim=True) * o.abs() + S * U * (pi @ va) + 17 * U * o.abs())
    return o, bound


# ------------------------------------------------------------------------------------- what test_fp32_grade_gpu runs
def split3_signature(src, out, seg=None, weight=False) -> tuple:
    return ("split3", "weight" if weight else "activation", "seg == cols" if (seg or src.shape[1]) == src.shape[1] else "seg < cols")


def softmax_signature(scores, n) -> tuple:
    return ("softmax_split3", "n == n_pad" if n == scores.shape[1] else "n < n_pad")


def attn_small_signature(qkv, out, heads) -> tuple:
    dense = qkv.stride(0) == 3 * heads * 64 and out.stride(0) == heads * 64
    return ("attn_small_f32", "dense strides" if dense else "padded strides")


SPLIT3_SEGS = ("cols", 128, 64)
SOFTMAX_N = (1, 2, 3, 4, 5, 63, 64, 65, 93, 2049, 32784)
ATTN_SEQS = (1, 31, 32, 33, 100, 257, 319, 320)
RUN_SIGNATURES = ({("split3", p, s) for p in ("activation", "weight") for s in ("seg == cols", "seg < cols")}
                  | {("softmax_split3", "n == n_pad"), ("softmax_split3", "n < n_pad")}
                  | {("attn_small_f32", "dense strides"), ("attn_small_f32", "padded strides")})


def pad64(n: int) -> int:
    return (n + 63) // 64 * 64


def check_bounded(got: torch.Tensor, exp: torch.Tensor, bound: torch.Tensor, what: str, ratios: dict, key: str) -> None:
    """kernel_exact.compare of an fp32 result against (exp, bound), keeping the largest |err| / bound under `key` (over
    the elements with a non-zero bound; compare has held the others to exactly zero error)."""
    kx.compare(got, exp, bound, what, store_rounding=False)
    err = (got.double() - exp).abs()
    r = float(torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.zeros_like(err)).max())
    ratios[key] = max(ratios.get(key, 0.0), r)
