"""The fp32-grade split-bf16 path element by element (-m gpu): split3, softmax_split3, attn_small_f32 and the GEMM on split
operands, at the shapes Stage II's vertex queries (autoencoder.py) and DinoV2's default precision (image_encoder.py) run.

split3 is bit-exact against the torch restatement of tests/split_exact.py; the split GEMMs are bit-exact on the exact
split grid in every role the pipeline uses them; softmax_split3, attn_small_f32 and the split GEMMs on real operands are
held to the per-element bounds derived there, up to Stage II's default window (Rp = 32 832 keys, K = 98 496 for P'V'^T)
and DinoV2-L over 16 frames.  Every output is a view into a NaN-filled buffer whose hidden elements must stay untouched,
and every input hides NaN past its last column.  The largest |error| / bound of every bounded check is printed at the end
of the module (pytest -s).
"""
import math

import pytest
import torch

import kernel_exact as kx
import split_exact as sx

pytestmark = pytest.mark.gpu
DEV = "cuda"
RATIOS: dict = {}


@pytest.fixture(scope="module")
def ops(amb_lib):
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from actionmesh_b200 import ops as o

    torch.cuda.reset_peak_memory_stats()
    yield o
    print("\nfp32-grade bounds, max |error| / bound:")
    for key, r in sorted(RATIOS.items()):
        print(f"  {key:40s} {r:.3g}")
    print(f"peak device memory: {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


def _nan_out(rows: int, cols: int, dtype, pad_cols: int = kx.PAD_COLS) -> tuple[torch.Tensor, torch.Tensor]:
    buf = kx.nan_buffer((rows + kx.PAD_ROWS, cols + pad_cols), dtype, DEV)
    return buf, buf[:rows, :cols]


def _untouched_after(buf: torch.Tensor, view: torch.Tensor, what: str) -> None:
    kx.int_view(view).fill_(kx.nan_bits(view.dtype))
    assert kx.is_untouched(buf), f"{what}: wrote outside its rows / columns"


# ------------------------------------------------------------------------------------------------------------- split3
def _split_inputs(rows: int, cols: int, gen: torch.Generator) -> torch.Tensor:
    """fp32 values of every kind, mixed element by element: normal values over 2^+-20, round-to-nearest ties
    (x = bf16 + exactly half a bf16 ulp), +0 and -0, values around 2^-126 (normal and subnormal), magnitudes up to 2^100."""
    shape = (rows, cols)
    kind = torch.randint(0, 6, shape, generator=gen, device=DEV)
    normal = torch.randn(shape, generator=gen, device=DEV) * torch.exp2(torch.randint(-20, 21, shape, generator=gen, device=DEV).float())
    b = torch.randn(shape, generator=gen, device=DEV).bfloat16().float()
    tie = b + torch.ldexp(torch.ones_like(b), torch.frexp(b)[1] - 9)
    zero = torch.zeros(shape, device=DEV)
    zero[torch.rand(shape, generator=gen, device=DEV) < 0.5] = -0.0
    tiny = torch.randn(shape, generator=gen, device=DEV) * 2.0 ** -126 * torch.exp2(torch.randint(-6, 3, shape, generator=gen, device=DEV).float())
    huge = torch.randn(shape, generator=gen, device=DEV) * torch.exp2(torch.randint(60, 101, shape, generator=gen, device=DEV).float())
    x = torch.stack([normal, tie, zero, tiny, huge, normal], -1).gather(-1, kind[..., None])[..., 0]
    return x.float()


@pytest.mark.parametrize("weight", [False, True], ids=["activation", "weight"])
@pytest.mark.parametrize("seg", sx.SPLIT3_SEGS)
def test_split3_is_bit_exact(ops, weight, seg):
    """Both patterns, one segment and segments of 128 and 64 columns, 1 / 37 / 4112 rows, with contiguous and with strided
    source and destination: every output bit equals the torch restatement, and |x - hi - lo| <= 2^-17 |x| + 2^-134."""
    cols = 256
    s = cols if seg == "cols" else seg
    gen = torch.Generator(device=DEV).manual_seed(17 + s + weight)
    for rows in (1, 37, 4112):
        for strided in (False, True):
            x = _split_inputs(rows, cols, gen)
            pc = kx.PAD_COLS if strided else 0
            _, src = kx.padded(x, pc, kx.PAD_ROWS)
            obuf, out = _nan_out(rows, 3 * cols, torch.bfloat16, pc + 8 if strided else 0)
            ops.split3(src, out, seg=s, weight=weight)
            what = f"split3 weight={weight} seg={s} rows={rows} strided={strided}"
            want = sx.split_layout(x.cpu(), s, weight)
            eq = kx.int_view(out.cpu()) == kx.int_view(want)
            assert bool(eq.all()), f"{what}: {int((~eq).sum())} elements differ from the restatement, first at {(~eq).nonzero()[0].tolist()}"
            hi, lo = sx.split_parts(x.cpu())
            err = (x.cpu().double() - hi.double() - lo.double()).abs()
            assert bool((err <= sx.SPLIT_REL * x.cpu().double().abs() + sx.SPLIT_ABS).all()), what
            _untouched_after(obuf, out, what)


def test_split3_returns_the_grid_parts(ops):
    gen = torch.Generator(device=DEV).manual_seed(3)
    for k in (128, 1024):
        x, hi, lo = sx.split_grid((300, k), k, gen, DEV)
        out = torch.empty(300, 3 * k, dtype=torch.bfloat16, device=DEV)
        ops.split3(x, out)
        assert torch.equal(out[:, :k].float(), hi) and torch.equal(out[:, k:2 * k].float(), lo) and torch.equal(out[:, 2 * k:].float(), hi)


# ---------------------------------------------------------------------------------------------------- softmax_split3
def _scores(rows: int, n: int, n_pad: int, gen: torch.Generator, scale: float) -> tuple[torch.Tensor, torch.Tensor]:
    """(buffer, view (rows, n_pad)): logits ~ N(0, 1) after scaling; every 4th row has its maximum in the last live
    column (the ragged float4 when n % 4 != 0), rows 2 mod 4 spread over 80 nats (maximum in the first column), rows
    3 mod 4 over 80 nats with the maximum last.  Padding columns hold NaN (even rows) or +1e30 (odd rows)."""
    y = torch.randn(rows, n, generator=gen, device=DEV)
    r = torch.arange(rows, device=DEV)
    spread = -80 * torch.rand(rows, n, generator=gen, device=DEV)
    y = torch.where((r % 4 >= 2)[:, None], spread, y)
    y[r % 4 == 0, n - 1] = 6.0
    y[r % 4 == 2, 0] = 0.5
    y[r % 4 == 3, n - 1] = 0.5
    x = (y / scale).float()
    buf = kx.nan_buffer((rows + kx.PAD_ROWS, n_pad + kx.PAD_COLS), torch.float32, DEV)
    buf[:rows, :n] = x
    pad = buf[:rows, n:n_pad]
    pad[1::2] = 1e30
    return buf, buf[:rows, :n_pad]


def _check_softmax(ops, rows: int, n: int, n_pad: int, seed: int) -> None:
    scale = 1.0 / math.sqrt(128)
    gen = torch.Generator(device=DEV).manual_seed(seed)
    sbuf, s = _scores(rows, n, n_pad, gen, scale)
    obuf, out = _nan_out(rows, 3 * n_pad, torch.bfloat16)
    ops.softmax_split3(s, n, scale, out)
    what = f"softmax_split3 rows={rows} n={n} n_pad={n_pad}"
    step = max(1, (1 << 25) // n_pad)
    for r0 in range(0, rows, step):
        r1 = min(rows, r0 + step)
        o = out[r0:r1]
        hi, lo, hi2 = o[:, :n_pad], o[:, n_pad:2 * n_pad], o[:, 2 * n_pad:]
        assert torch.equal(kx.int_view(hi2), kx.int_view(hi)), f"{what}: third part differs from the first"
        assert bool((kx.int_view(o.view(r1 - r0, 3, n_pad)[:, :, n:]) == 0).all()), f"{what}: padding columns are not +0"
        hf, lf = hi[:, :n].double(), lo[:, :n].double()
        assert bool((lf.abs() <= kx.half_ulp_bf16(hf)).all()), f"{what}: |p_lo| above half a bf16 ulp of p_hi"
        p64, bound = sx.softmax_bound(s[r0:r1, :n], scale)
        sx.check_bounded(hf + lf, p64, bound, f"{what} rows [{r0}, {r1})", RATIOS, f"softmax_split3 n={n}")
    _untouched_after(obuf, out, what)
    assert kx.is_untouched(sbuf[:, n_pad:]) and kx.is_untouched(sbuf[rows:])


@pytest.mark.parametrize("n", sx.SOFTMAX_N)
def test_softmax_split3(ops, n):
    """n_pad = pad64(n) and n_pad well past it, on 1, 5 and 16 384 rows (16 384 x 32 832 is Stage II's production chunk)."""
    for rows in (1, 5, 16384):
        for n_pad in (sx.pad64(n), sx.pad64(n) + 4 * 64 + 4):
            _check_softmax(ops, rows, n, n_pad, seed=n + rows + n_pad)
    torch.cuda.empty_cache()


# ----------------------------------------------------------------------------------------------------- attn_small_f32
def _attn_qkv(frames: int, seq: int, heads: int, gen: torch.Generator, padded: bool):
    """fp32 qkv (frames seq, 3 heads 64) and out views; q, k ~ N(0, 1), v ~ U[0.5, 1.5); every 7th query row is scaled by
    20 (a logit spread of tens of nats)."""
    D = heads * 64
    M = frames * seq
    q = torch.randn(M, D, generator=gen, device=DEV)
    q[::7] *= 20
    k = torch.randn(M, D, generator=gen, device=DEV)
    v = torch.rand(M, D, generator=gen, device=DEV) + 0.5
    vals = torch.cat([q, k, v], 1)
    pc = kx.PAD_COLS if padded else 0
    qbuf, qkv = kx.padded(vals, pc, kx.PAD_ROWS)
    obuf, out = _nan_out(M, D, torch.float32, pc)
    return qbuf, qkv, obuf, out


def _check_attn(qkv, out, frames, seq, heads, scale, what):
    D = heads * 64
    per = lambda t: t.view(frames, seq, heads, 64).permute(0, 2, 1, 3).reshape(frames * heads, seq, 64)
    q, k, v = per(qkv[:, :D].contiguous()), per(qkv[:, D:2 * D].contiguous()), per(qkv[:, 2 * D:].contiguous())
    o64, bound = sx.attn_small_bound(q, k, v, scale)
    sx.check_bounded(per(out.contiguous()), o64, bound, what, RATIOS, f"attn_small_f32 seq={seq}")


@pytest.mark.parametrize("seq", sx.ATTN_SEQS)
def test_attn_small_f32(ops, seq):
    """Every element within the bound, with padded row strides (NaN canaries past q / k / v and the output) and dense."""
    scale = 1.0 / 8
    for padded, frames, heads in ((True, 3, 2), (False, 2, 3)):
        gen = torch.Generator(device=DEV).manual_seed(seq + padded)
        qbuf, qkv, obuf, out = _attn_qkv(frames, seq, heads, gen, padded)
        ops.attn_small_f32(qkv, frames, seq, heads, scale, out)
        what = f"attn_small_f32 seq={seq} padded={padded}"
        _check_attn(qkv, out, frames, seq, heads, scale, what)
        _untouched_after(obuf, out, what)


def test_attn_small_f32_dinov2_l(ops):
    """DinoV2-L's call (16 frames x 16 heads x 257 tokens) within the bound; one frame run alone equals its slice of the
    full call bit for bit."""
    frames, seq, heads, scale = 16, 257, 16, 1.0 / 8
    gen = torch.Generator(device=DEV).manual_seed(257)
    _, qkv, obuf, out = _attn_qkv(frames, seq, heads, gen, False)
    ops.attn_small_f32(qkv, frames, seq, heads, scale, out, tag="attn_dino")
    _check_attn(qkv, out, frames, seq, heads, scale, "attn_small_f32 DinoV2-L")
    for f in (0, 11, 15):
        _, o1 = _nan_out(seq, heads * 64, torch.float32)
        ops.attn_small_f32(qkv[f * seq:(f + 1) * seq], 1, seq, heads, scale, o1)
        assert torch.equal(kx.int_view(o1), kx.int_view(out[f * seq:(f + 1) * seq])), f"frame {f} alone differs"
    _untouched_after(obuf, out, "attn_small_f32 DinoV2-L")


# -------------------------------------------------------------------------------------------- split GEMMs, exact grid
def _split(ops, x: torch.Tensor, seg=None, weight=False) -> torch.Tensor:
    """split3 of x into a view of a NaN-filled buffer with hidden columns (the GEMM's operands hide NaN past K)."""
    rows, cols = x.shape
    _, src = kx.padded(x, kx.PAD_COLS)
    _, out = _nan_out(rows, 3 * cols, torch.bfloat16)
    return ops.split3(src, out, seg=seg, weight=weight)


def _exact(a_hi, a_lo, w_hi, w_lo) -> torch.Tensor:
    """fp64 sum of a_hi w_hi + a_lo w_hi + a_hi w_lo: the exact product minus the dropped lo lo term."""
    a, w = (a_hi + a_lo).double(), (w_hi + w_lo).double()
    return a @ w.t() - a_lo.double() @ w_lo.double().t()


@pytest.mark.parametrize("m,n,k", [(1, 256, 128), (129, 256, 128), (640, 192, 128), (300, 256, 1024), (129, 1024, 1024)],
                         ids=["m1_bn128", "m129_bn128", "m640_bn64", "coop_k3072", "coop_n1024"])
def test_split_gemm_activation_weight_exact(ops, m, n, k):
    """Activation x weight ([hi|lo|hi] x [hi|hi|lo]) on ping-pong BN = 128 and 64 tiles and on the cooperative tiles
    (K' = 3072): bit for bit."""
    gen = torch.Generator(device=DEV).manual_seed(m + n + k)
    a, a_hi, a_lo = sx.split_grid((m, k), k, gen, DEV)
    w, w_hi, w_lo = sx.split_grid((n, k), k, gen, DEV)
    obuf, out = _nan_out(m, n, torch.float32)
    ops.gemm(_split(ops, a), _split(ops, w, weight=True), out)
    kx.compare(out, _exact(a_hi, a_lo, w_hi, w_lo), None, f"split gemm {m}x{n}x{k}")
    _untouched_after(obuf, out, "split gemm")


def test_split_gemm_per_head_scores_exact(ops):
    """The score GEMM's operands: q3 = split3(q, seg = 128) and k3 = split3(k, seg = 128, weight), one head's 384-column
    slice of each (autoencoder.py), N = 320 keys on BN = 64 tiles: bit for bit, every head."""
    m, keys, H, dh = 300, 320, 4, 128
    gen = torch.Generator(device=DEV).manual_seed(5)
    q, q_hi, q_lo = sx.split_grid((m, H * dh), dh, gen, DEV)
    kk, k_hi, k_lo = sx.split_grid((keys, H * dh), dh, gen, DEV)
    q3, k3 = _split(ops, q, seg=dh), _split(ops, kk, seg=dh, weight=True)
    for h in range(H):
        obuf, out = _nan_out(m, keys, torch.float32, 0)
        c = slice(h * 3 * dh, (h + 1) * 3 * dh)
        ops.gemm(q3[:, c], k3[:, c], out)
        d = slice(h * dh, (h + 1) * dh)
        kx.compare(out, _exact(q_hi[:, d], q_lo[:, d], k_hi[:, d], k_lo[:, d]), None, f"scores head {h}")
        _untouched_after(obuf, out, f"scores head {h}")


def test_split_gemm_weight_as_a_operand_exact(ops):
    """V-transpose: the weight split [hi|hi|lo] as the A operand against [hi|lo|hi] activations (V^T = W_v ctx^T,
    K' = 3072, N = Rp = 320 on BN = 64 tiles): the products are w_hi c_hi + w_hi c_lo + w_lo c_hi, bit for bit."""
    D, Rp = 1024, 320
    gen = torch.Generator(device=DEV).manual_seed(6)
    wv, w_hi, w_lo = sx.split_grid((D, D), D, gen, DEV)
    ctx, c_hi, c_lo = sx.split_grid((Rp, D), D, gen, DEV)
    obuf, out = _nan_out(D, Rp, torch.float32, 0)
    ops.gemm(_split(ops, wv, weight=True), _split(ops, ctx), out)
    kx.compare(out, _exact(w_hi, w_lo, c_hi, c_lo), None, "V-transpose")
    _untouched_after(obuf, out, "V-transpose")


def test_split_gemm_pv_exact_at_production_depth(ops):
    """P'V'^T at Stage II's default window (R = 32 784 keys, Rp = 32 832, K' = 98 496): scores in {0, -1e4} with a power
    of two c of live zeros per row make softmax_split3 write p = 1/c exactly (p_lo = 0, padding 0), so the product with
    grid-valued V^T is exact; the output is a head's 128 columns of a 1024-wide buffer.  Bit for bit."""
    R, Rp, m, dh, D = 32784, 32832, 300, 128, 1024
    scale = 1.0 / math.sqrt(dh)
    gen = torch.Generator(device=DEV).manual_seed(7)
    c = 2 ** torch.randint(0, 7, (m,), generator=gen, device=DEV)
    mask = torch.rand(m, R, generator=gen, device=DEV).argsort(-1) < c[:, None]   # c random live keys per row
    odd = torch.arange(m, device=DEV) % 2 == 1                                      # odd rows: the last key is live
    move = (odd & ~mask[:, R - 1]).nonzero()[:, 0]
    mask[move, mask[move].int().argmax(-1)] = False
    mask[move, R - 1] = True
    sbuf = kx.nan_buffer((m, Rp + kx.PAD_COLS), torch.float32, DEV)
    sbuf[:, :R] = torch.where(mask, 0.0, -1e4)
    _, p3 = _nan_out(m, 3 * Rp, torch.bfloat16)
    ops.softmax_split3(sbuf[:, :Rp], R, scale, p3)
    P = mask.double() / c[:, None].double()
    assert torch.equal(p3[:, :R].double(), P) and torch.equal(p3[:, 2 * Rp:2 * Rp + R].double(), P)
    assert bool((kx.int_view(p3[:, Rp:2 * Rp]) == 0).all()) and bool((kx.int_view(p3.view(m, 3, Rp)[:, :, R:]) == 0).all())
    vt, _, _ = sx.split_grid((dh, Rp), 128, gen, DEV)   # the bit budget holds: at most 64 live terms of 1/c
    obuf, o = _nan_out(m, D, torch.float32)
    out = o[:, 3 * dh:4 * dh]
    ops.gemm(p3, _split(ops, vt, weight=True), out)
    kx.compare(out, P @ vt[:, :R].double().t(), None, "P'V'^T exact")
    _untouched_after(obuf, out, "P'V'^T exact")


# ------------------------------------------------------------------------------------ split GEMMs, production shapes
def _check_split_gemm(out, a, w, what, key, chunk=2048, **epi):
    """Every element of out (rows of a x rows of w) against split_exact's bound plus the epilogue, in row chunks."""
    for r0 in range(0, a.shape[0], chunk):
        r1 = min(a.shape[0], r0 + chunk)
        c64, b = sx.split_gemm_bound(a[r0:r1], w)
        e = {name: (v[r0:r1] if name == "residual" and v is not None else v) for name, v in epi.items()}
        v, bound = sx.epilogue_bound(c64, b, **e)
        sx.check_bounded(out[r0:r1], v, bound, f"{what} rows [{r0}, {r1})", RATIOS, key)


def _weight(n, k, gen):
    return torch.randn(n, k, generator=gen, device=DEV) / math.sqrt(k)


def test_stage2_query_attention_production(ops):
    """Stage II at the default window (V chunk 16 384, D 1024, H 8, R = 32 784, Rp = 32 832), one head: the score GEMM
    (BN = 64, N = 32 832, K' = 384), V-transpose (1024 x 32 832, K' = 3072) and P'V'^T (K' = 98 496, strided fp32 output)
    on the softmax_split3 output.  V^T for P'V'^T is U[0.5, 1.5): one sign, so the accumulation errors add up."""
    Vc, D, dh, R, Rp = 16384, 1024, 128, 32784, 32832
    scale = 1.0 / math.sqrt(dh)
    gen = torch.Generator(device=DEV).manual_seed(11)
    q = torch.randn(Vc, dh, generator=gen, device=DEV)
    k = torch.randn(Rp, dh, generator=gen, device=DEV)
    k[R:] = 0                                          # pad rows of ctx are zero: K rows of zeros
    sbuf, s32 = _nan_out(Vc, Rp, torch.float32, 0)
    ops.gemm(_split(ops, q, seg=dh), _split(ops, k, seg=dh, weight=True), s32, tag="s2_q")
    _check_split_gemm(s32, q, k, "score GEMM", "score GEMM K'=384", chunk=1024)
    _, p3 = _nan_out(Vc, 3 * Rp, torch.bfloat16)
    ops.softmax_split3(s32, R, scale, p3)
    del sbuf, s32
    torch.cuda.empty_cache()
    # V-transpose: W_v (D, D) as the A operand against ctx (Rp, D)
    wv = _weight(D, D, gen)
    ctx = torch.randn(Rp, D, generator=gen, device=DEV)
    ctx[R:] = 0
    vbuf, vt32 = _nan_out(D, Rp, torch.float32, 0)
    ops.gemm(_split(ops, wv, weight=True), _split(ops, ctx), vt32, tag="s2_q")
    _check_split_gemm(vt32, wv, ctx, "V-transpose", "V-transpose K'=3072", chunk=256)
    del vbuf, vt32, ctx
    # P'V'^T: one head's 128 columns of the (Vc, D) output
    vt = torch.rand(dh, Rp, generator=gen, device=DEV) + 0.5
    vt[:, R:] = 0
    vt3 = _split(ops, vt, weight=True)
    obuf, o = _nan_out(Vc, D, torch.float32)
    out = o[:, 5 * dh:6 * dh]
    ops.gemm(p3, vt3, out, tag="s2_q")
    for r0 in range(0, Vc, 2048):
        p = p3[r0:r0 + 2048, :Rp].double() + p3[r0:r0 + 2048, Rp:2 * Rp].double()
        c64, b = sx.split_gemm_bound(p, vt)
        sx.check_bounded(out[r0:r0 + 2048], c64, b, f"P'V'^T rows [{r0}, {r0 + 2048})", RATIOS, "P'V'^T K'=98496")
    _untouched_after(obuf, out, "P'V'^T")


def _ls_case(ops, m, n, k, gen, *, act=0, col_scale=False, residual=False, a_kind="normal"):
    a = torch.randn(m, k, generator=gen, device=DEV) if a_kind == "normal" else \
        kx.gelu64(torch.randn(m, k, generator=gen, device=DEV).double()).float()
    w = _weight(n, k, gen)
    bias = kx.padded_vector(torch.randn(n, generator=gen, device=DEV) * 0.1)
    kw = dict(bias=bias)
    if act:
        kw["act"] = act
    if col_scale:
        kw["col_scale"] = kx.padded_vector(torch.rand(n, generator=gen, device=DEV) + 0.05)
    obuf, out = _nan_out(m, n, torch.float32)
    res = None
    if residual:
        res = torch.randn(m, n, generator=gen, device=DEV)
        out.copy_(res)
        kw["residual"] = out
    ops.gemm(_split(ops, a), _split(ops, w, weight=True), out, **kw)
    epi = dict(bias=bias, act=act, col_scale=kw.get("col_scale"), residual=res)
    return obuf, out, a, w, epi


@pytest.mark.parametrize("name,m,n,k,act,ls,res,a_kind", [
    ("stage2_ff2_res", 16384, 1024, 4096, 0, False, True, "gelu"),
    ("dinov2l_qkv", 16 * 257, 3072, 1024, 0, False, False, "normal"),
    ("dinov2l_ff1_gelu", 16 * 257, 4096, 1024, 1, False, False, "normal"),
    ("dinov2l_ff2_ls_res", 16 * 257, 1024, 4096, 0, True, True, "gelu"),
])
def test_split_gemm_production_epilogues(ops, name, m, n, k, act, ls, res, a_kind):
    """The cooperative split GEMMs (N a multiple of 256, K' = 3072 or 12 288) with their epilogues, every element."""
    gen = torch.Generator(device=DEV).manual_seed(m + n + k)
    obuf, out, a, w, epi = _ls_case(ops, m, n, k, gen, act=act, col_scale=ls, residual=res, a_kind=a_kind)
    _check_split_gemm(out, a, w, name, f"{name} K'={3 * k}", chunk=1024, **epi)
    _untouched_after(obuf, out, name)
    del obuf, out, a, w, epi
    torch.cuda.empty_cache()
