"""The C-ABI entry points outside the GEMM and attention (-m gpu), each against an fp64 torch restatement, element by element.

Bounds are derived from the kernels' fp32 operations (u = 2^-24, the unit roundoff of fp32; expf / sinf / cosf / rsqrtf
are within 2 ulp, i.e. 4u relative for expf and rsqrtf and 4u absolute for sinf / cosf of results in [-1, 1]); a bf16
output adds half a bf16 ulp.  Strided operands and outputs are views into NaN-filled buffers (tests/kernel_exact.py), and
what a kernel must not write has to keep its NaN bits.
"""
import math

import pytest
import torch

import kernel_exact as kx

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = kx.U


@pytest.fixture(scope="module")
def ops(amb_lib):
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from actionmesh_b200 import ops as o

    return o


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


# ------------------------------------------------------------------------------------------------------- LayerNorm
def _lane_order_stats(x: torch.Tensor, cols: int) -> tuple[torch.Tensor, torch.Tensor]:
    """The kernel's fp32 statistics in its order: lane l sums its elements (j * 32 + l) * 8 + t for j, t in turn, the 32
    lane sums are combined by an xor butterfly (16, 8, 4, 2, 1), and the centred squares are summed the same way with
    q += d * d contracted to one rounding."""
    per_lane = cols // 32
    v = x.float().view(-1, cols // 256, 32, 8).permute(0, 2, 1, 3).reshape(-1, 32, per_lane)

    def lane_sum(terms, fused):
        s = torch.zeros(terms.shape[:2], dtype=torch.float32, device=x.device)
        for j in range(per_lane):
            s = (s.double() + terms[..., j].double() ** 2).float() if fused else s + terms[..., j]
        lane = torch.arange(32, device=x.device)
        for o in (16, 8, 4, 2, 1):
            s = s + s[:, lane ^ o]
        return s[:, 0]

    mean = lane_sum(v, False) * (1.0 / cols)
    q = lane_sum(v - mean[:, None, None], True)
    return mean, q


@pytest.mark.parametrize("cols", [256, 512, 1024, 2048, 4096])
@pytest.mark.parametrize("x_dt,y_dt", [(torch.bfloat16, torch.bfloat16), (torch.float32, torch.bfloat16),
                                       (torch.bfloat16, torch.float32), (torch.float32, torch.float32)])
def test_layernorm(ops, cols, x_dt, y_dt):
    """Against the fp64 normalisation of the kernel's own fp32 mean and centred sum of squares (restated in its order by
    _lane_order_stats): rstd = rsqrtf(q / cols + eps) is within 2 ulp plus the rounding of the sum, and the fp32 products
    (x - mean) * rstd * g + b add 3 roundings, so |d| <= (8 + cols / 64) u |(x - mean) rstd g| + u |y|.  Fp32 rows with mean
    1e3 and std 1e-2 are included: a one-pass variance E[x²] - E[x]² cancels 1e6 against 1e6 there and fails."""
    g = _gen(cols)
    rows = 203
    x = torch.randn(rows, cols, generator=g, device=DEV) * 3 + 0.5
    if x_dt == torch.float32:
        x[::7] = 1e3 + torch.randn(x[::7].shape, generator=g, device=DEV) * 1e-2
    x = x.to(x_dt)
    _, xv = kx.padded(x, 24, 2)
    gamma = kx.padded_vector(torch.randn(cols, generator=g, device=DEV))
    beta = kx.padded_vector(torch.randn(cols, generator=g, device=DEV))
    ybuf = kx.nan_buffer((rows + 2, cols + 40), y_dt, DEV)
    y = ybuf[:rows, :cols]
    ops.layernorm(xv, gamma, beta, 1e-5, out=y)
    mean, q = _lane_order_stats(x, cols)
    rstd = 1.0 / torch.sqrt(q.double() / cols + float(torch.tensor(1e-5)))
    xhat = (x.float() - mean[:, None]).double() * rstd[:, None] * gamma.double()
    want = xhat + beta.double()
    bound = (8 + cols / 64) * U * xhat.abs() + U * want.abs()
    kx.compare(y, want, bound, f"layernorm {cols} {x_dt}->{y_dt}")
    kx.int_view(y).fill_(kx.nan_bits(y_dt))
    assert kx.is_untouched(ybuf)


# ------------------------------------------------------------------------------------------------- cfg_euler_step
@pytest.mark.parametrize("n_branches", [1, 2, 3, 4])
def test_cfg_euler_step(ops, n_branches):
    """x += dt (p_0 + sum_i s_i (p_i - p_(i-1))) on updated frames: differences of bf16 values are exact in fp32, each
    fused multiply-add rounds once by u of its partial sum (<= V = |p_0| + sum_i |s_i (p_i - p_(i-1))|), and the final
    x + dt v once more: |d| <= u (|x'| + n |dt| V).  Observed frames come back bit-identical."""
    g = _gen(40 + n_branches)
    F, N, C = 6, 37, 64
    n_per = N * C
    x0 = torch.randn(F, n_per, generator=g, device=DEV)
    pred = torch.randn(n_branches, F, N + 1, C, generator=g, device=DEV).bfloat16()  # row 0 of a frame: time token
    upd = torch.tensor([1, 0, 1, 1, 0, 1], dtype=torch.uint8, device=DEV)
    scales = [7.5, -2.25, 3.0][:n_branches - 1]
    dt = -0.0625
    x = x0.clone()
    ops.cfg_euler_step(x, pred, scales, dt, upd, n_branches=n_branches, branch_stride=F * (N + 1) * C, frame_stride=(N + 1) * C,
                       frame_offset=C, n_per_frame=n_per)
    p = pred[:, :, 1:].reshape(n_branches, F, n_per).double()
    v, V = p[0].clone(), p[0].abs()
    for i in range(1, n_branches):
        v = v + scales[i - 1] * (p[i] - p[i - 1])
        V = V + abs(scales[i - 1]) * (p[i] - p[i - 1]).abs()
    want = x0.double() + dt * v
    bound = U * (want.abs() + n_branches * abs(dt) * V)
    m = upd.bool()
    kx.compare(x[m], want[m], bound[m], f"cfg_euler_step {n_branches} branches")
    assert torch.equal(kx.int_view(x[~m]), kx.int_view(x0[~m]))


# ------------------------------------------------------------------------------------------- sinusoidal embeddings
def _sincos_bound(a):
    """fp32 frequencies w = expf(-ln(1e4) j / half): the argument rounds twice (and the constant once) on |arg| <= 9.22,
    expf adds 4u: w is within 27u relative, a = t w within 28u; sinf / cosf add 4u absolute."""
    return 28 * U * a.abs() + 4 * U


def test_timestep_embedding_with_mask(ops):
    g = _gen(50)
    B, T, ch = 3, 5, 256
    t = torch.rand(B, generator=g, device=DEV) * 1000
    mask = (torch.rand(B * T, generator=g, device=DEV) < 0.4).float()
    out = ops.timestep_embedding(t, ch, mask=mask)
    half = ch // 2
    tv = t.double()[torch.arange(B * T, device=DEV) % B] * (1 - mask.double())
    w = torch.exp(-math.log(1e4) * torch.arange(half, device=DEV, dtype=torch.float64) / half)
    a = tv[:, None] * w[None]
    want = torch.cat([a.sin(), a.cos()], 1)
    bound = torch.cat([_sincos_bound(a)] * 2, 1)
    kx.compare(out, want, bound, "timestep_embedding")
    masked = mask.bool()
    assert torch.equal(out[masked, :half].float(), torch.zeros_like(out[masked, :half].float()))  # t = 0: sin 0, cos 1
    assert bool((out[masked, half:] == 1).all())


def test_alpha_rows(ops):
    size, rows = 256, 7
    buf = kx.nan_buffer((rows + 2, 2 * size + 24), torch.float32, DEV)
    view = buf[:rows, :2 * size]
    src, tgt = 0.3, 0.85
    ops.alpha_rows(src, tgt, size, view)
    half = size // 2
    w = torch.exp(-math.log(1e4) * torch.arange(half, device=DEV, dtype=torch.float64) / half)
    parts, bounds = [], []
    for s in (float(torch.tensor(src)), float(torch.tensor(tgt))):
        a = s * w
        parts += [a.cos(), a.sin()]
        bounds += [_sincos_bound(a)] * 2
    want, bound = torch.cat(parts)[None].expand(rows, -1), torch.cat(bounds)[None].expand(rows, -1)
    kx.compare(view, want, bound, "alpha_rows")
    kx.int_view(view).fill_(kx.NAN_F32)
    assert kx.is_untouched(buf)


@pytest.mark.parametrize("include_pi", [False, True])
def test_point_embedding(ops, include_pi):
    """x and the extra features are copied and the padding is zero (bit-exact); a = x * (2^f [* fp32 pi]) rounds once
    (u |a|) and sinf / cosf add 4u."""
    g = _gen(60)
    V, E, F, kpad = 1000, 2, 8, 64
    pts = torch.rand(V, 3 + E, generator=g, device=DEV) * 2 - 1
    out = ops.point_embedding(pts, F, include_pi, kpad)
    fr = 2.0 ** torch.arange(F, device=DEV, dtype=torch.float64)
    if include_pi:
        fr = fr * float(torch.tensor(math.pi, dtype=torch.float32))
    a = (pts[:, :3].double()[:, :, None] * fr).reshape(V, 3 * F)
    bound = U * a.abs() + 4 * U
    kx.compare(out[:, 3:3 + 3 * F], a.sin(), bound, "point_embedding sin")
    kx.compare(out[:, 3 + 3 * F:3 + 6 * F], a.cos(), bound, "point_embedding cos")
    assert torch.equal(out[:, :3], pts[:, :3])
    assert torch.equal(out[:, 3 + 6 * F:3 + 6 * F + E], pts[:, 3:])
    assert bool((out[:, 3 + 6 * F + E:] == 0).all())


def test_displacement_out(ops):
    """y = 2 / (1 + expf(-x)) - 1 with x = -logit: expf 4u, the sum and the correctly rounded division u each, so q = 2 / (1 +
    e) is within 6u |q|, and the subtraction adds u |y|."""
    g = _gen(70)
    V, ld, od = 777, 64, 3
    _, logits = kx.padded(torch.randn(V, od, generator=g, device=DEV) * 4, ld - od)
    out = torch.empty(V, od, device=DEV)
    ops.displacement_out(logits, od, out)
    q = 2 / (1 + torch.exp(logits.double()))
    want = q - 1
    kx.compare(out, want, 6 * U * q.abs() + U * want.abs(), "displacement_out")


@pytest.mark.parametrize("which", ["z,logvar,std", "z", "logvar", "std", "logvar,std"])
def test_gaussian_sample(ops, which):
    """logvar = clamp(params[:, C:2C], -30, 20) is exact; std = expf(logvar / 2) is within 4u; z = mean + std * eps with
    explicitly rounded product and sum: |d| <= u |z| + 5u |std eps|.  Outputs not passed stay unwritten (NULL)."""
    g = _gen(80)
    rows, C, ld = 300, 64, 136
    _, params = kx.padded(torch.randn(rows, 2 * C, generator=g, device=DEV) * 12, ld - 2 * C)
    eps = torch.randn(rows, C, generator=g, device=DEV)
    outs = {k: torch.full((rows, C), float("nan"), device=DEV) for k in which.split(",")}
    ops.gaussian_sample(params, eps if "z" in outs else None, **outs)
    lv = params[:, C:].double().clamp(-30, 20)
    sd = torch.exp(0.5 * lv)
    if "logvar" in outs:
        assert torch.equal(outs["logvar"].double(), lv)
    if "std" in outs:
        kx.compare(outs["std"], sd, 4 * U * sd, "gaussian_sample std")
    if "z" in outs:
        z = params[:, :C].double() + sd * eps.double()
        kx.compare(outs["z"], z, U * z.abs() + 5 * U * (sd * eps.double()).abs(), "gaussian_sample z")


def test_patchify_is_unfold(ops):
    """im2col of the pixels, bit for bit: rows (t, py, px), columns (c, ky, kx) as unfold orders them, zeros up to kpad."""
    g = _gen(90)
    T, H, W, P, kpad = 3, 42, 56, 14, 640
    pix = torch.randn(T, 3, H, W, generator=g, device=DEV)
    out = ops.patchify(pix, P, kpad)
    cols = torch.nn.functional.unfold(pix, P, stride=P).transpose(1, 2).reshape(-1, 3 * P * P)
    want = torch.zeros(cols.shape[0], kpad, device=DEV)
    want[:, :3 * P * P] = cols
    assert torch.equal(kx.int_view(out), kx.int_view(want.bfloat16()))
