"""Exact restatements of ActionBench's metric kernels, for the bit-for-bit tests (not collected by pytest).

`csrc/icp.cu` rounds every fp32 operation explicitly (__fmul_rn, __fmaf_rn, __fadd_rn, __fsub_rn) and `csrc/chamfer.cu`
is built without fast math, so each fp32 result is one correctly rounded operation and can be restated here operation
for operation.  The fp64 sums of icp.cu are exact term by term (an fp32 difference squared, or times an fp32
coordinate, fits in 53 bits) and are added in a fixed order with no atomics; the restatement adds them in that order.
The nearest-neighbour kernels keep the first minimum (strict `<` in index order, or a 64-bit atomicMin on
(d² bits, index)), which is `torch.argmin`'s first minimum.

Only elementwise torch ops are used (no matmul, cdist or reductions whose order torch picks, except argmin), so the
helpers run on CPU tensors and, chunked, on CUDA ones.

fp32 additions, products and differences are torch's fp32 ops, which round correctly.  An fp32 fused multiply-add is
`fma32`: the product is exact in fp64, the sum is rounded to odd in fp64 (TwoSum gives the error) and then to fp32;
rounding to odd with 29 spare bits makes the second rounding correct, where plain fp64 rounding may double-round.
"""
from __future__ import annotations

import torch

# csrc/icp.cu: threads per block, and gt points per gt->pred thread.  The block sums below follow this layout.
ICP_THREADS = 128
ICP_QB = 4
NN_CHUNK = 1 << 24          # query x reference pairs per chunk of `nearest`


def fma32(a: torch.Tensor, b: torch.Tensor, c: torch.Tensor) -> torch.Tensor:
    """fp32 fmaf(a, b, c), correctly rounded (fp32 tensors of broadcastable shapes)."""
    p = a.double() * b.double()                 # exact: 24 + 24 bits
    c = c.double()
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)             # TwoSum: s + err == p + c exactly
    even = (s.view(torch.int64) & 1) == 0
    toward = torch.where(err > 0, torch.full_like(s, float("inf")), torch.full_like(s, float("-inf")))
    s = torch.where((err != 0) & even, torch.nextafter(s, toward), s)
    return s.float()


def naive_fma32(a: torch.Tensor, b: torch.Tensor, c: torch.Tensor) -> torch.Tensor:
    """float(a * b + c) in fp64: double-rounds on midpoint cases (kept to show that fma32 is needed)."""
    return (a.double() * b.double() + c.double()).float()


def icp_transform(x: torch.Tensor, R: torch.Tensor, s: torch.Tensor, T: torch.Tensor) -> torch.Tensor:
    """icp.cu::icp_transform: y_l = fl(fma(c, R[2][l], fma(b, R[1][l], fl(a R[0][l]))) + T_l), (a, b, c) = fl(s ⊙ x).
    x (..., 3), R (..., 3, 3), s and T (..., 3), broadcast against each other."""
    a, b, c = s[..., 0] * x[..., 0], s[..., 1] * x[..., 1], s[..., 2] * x[..., 2]
    ys = [fma32(c, R[..., 2, l], fma32(b, R[..., 1, l], a * R[..., 0, l])) + T[..., l] for l in range(3)]
    return torch.stack(ys, -1)


def dist2(p: torch.Tensor, q: torch.Tensor) -> torch.Tensor:
    """icp.cu::icp_dist2 and chamfer.cu's distance: fma(dz, dz, fma(dy, dy, fl(dx dx))), d = fl(p - q)."""
    dx, dy, dz = p[..., 0] - q[..., 0], p[..., 1] - q[..., 1], p[..., 2] - q[..., 2]
    return fma32(dz, dz, fma32(dy, dy, dx * dx))


def nearest(query: torch.Tensor, ref: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """(M, 3), (N, 3) fp32 -> (squared distance (M,) fp32, index (M,) int64) of each query's nearest reference point, the
    lowest index among equal minima.  Chunked over the queries."""
    n = ref.shape[0]
    step = max(1, NN_CHUNK // max(n, 1))
    ds, idx = [], []
    for q0 in range(0, query.shape[0], step):
        d = dist2(query[q0:q0 + step, None, :], ref[None])
        i = d.argmin(1)
        ds.append(d.gather(1, i[:, None])[:, 0])
        idx.append(i)
        del d
    return torch.cat(ds), torch.cat(idx)


def nn_distance(d2: torch.Tensor) -> torch.Tensor:
    """chamfer.cu's sqrtf of the squared distance: the fp64 root rounded to fp32 (a double rounding that cannot change a
    square root)."""
    return d2.double().sqrt().float()


def warp_tree(a: torch.Tensor) -> torch.Tensor:
    """Lane 0 of `a += __shfl_down_sync(~0, a, o)` for o = 16, 8, 4, 2, 1 over the lanes of dim -2 (size 32)."""
    for o in (16, 8, 4, 2, 1):
        a = a[..., :o, :] + a[..., o:2 * o, :]
    return a[..., 0, :]


def block_sum(v: torch.Tensor) -> torch.Tensor:
    """icp.cu::icp_block_store: (..., ICP_THREADS, k) per-thread values -> (..., k): the shuffle tree in every warp, then
    0.0 + w0 + w1 + w2 + w3 in warp order."""
    w = warp_tree(v.reshape(*v.shape[:-2], ICP_THREADS // 32, 32, v.shape[-1]))
    out = torch.zeros_like(w[..., 0, :])
    for k in range(ICP_THREADS // 32):
        out = out + w[..., k, :]
    return out


def contribution(x: torch.Tensor, y: torch.Tensor, g: torch.Tensor) -> torch.Tensor:
    """icp.cu::icp_contribution: (..., 3) fp32 -> (..., 13) fp64 = |e|², e, x ⊗ e (x index first), e = fl(y - g)."""
    e = (y - g).double()
    xs = x.double()
    v0 = (e[..., 0] * e[..., 0] + e[..., 1] * e[..., 1]) + e[..., 2] * e[..., 2]
    return torch.cat([v0[..., None], e, (xs[..., :, None] * e[..., None, :]).flatten(-2)], -1)


def _pad(v: torch.Tensor, n: int) -> torch.Tensor:
    return torch.cat([v, v.new_zeros(*v.shape[:-2], n - v.shape[-2], v.shape[-1])], -2)


def _in_order(slots: torch.Tensor) -> torch.Tensor:
    out = torch.zeros_like(slots[..., 0, :])
    for k in range(slots.shape[-2]):
        out = out + slots[..., k, :]
    return out


def icp_nearest(x: torch.Tensor, g: torch.Tensor, rot: torch.Tensor, params: torch.Tensor):
    """Both directions' nearest neighbours of every candidate: y (C, P, 3), a (C, P) into g, b (C, Q) into x."""
    y = icp_transform(x[None], rot[:, None], params[:, None, 9:], params[:, None, :3])
    C, P = y.shape[:2]
    a = nearest(y.reshape(C * P, 3), g)[1].reshape(C, P)
    b = torch.stack([nearest(g, y[n])[1] for n in range(C)])
    return y, a, b


def icp_sums(x: torch.Tensor, g: torch.Tensor, rot: torch.Tensor, params: torch.Tensor) -> torch.Tensor:
    """amb_icp_chamfer_grad of one frame: x (P, 3), g (Q, 3), rot (C, 3, 3), params (C, 12) fp32 -> (C, 13) fp64, summed
    in the kernel's order."""
    P, Q = x.shape[0], g.shape[0]
    y, a, b = icp_nearest(x, g, rot, params)
    C = y.shape[0]
    # pred -> gt: thread t of tile p owns point 128 p + t; threads past P add zeros
    tiles_p = (P + ICP_THREADS - 1) // ICP_THREADS
    v = _pad(contribution(x[None].expand(C, P, 3), y, g[a]), tiles_p * ICP_THREADS)
    s_pg = _in_order(block_sum(v.reshape(C, tiles_p, ICP_THREADS, 13)))
    # gt -> pred: thread t of tile q adds gt points (ICP_QB q + u) 128 + t for u = 0..3, in order, from 0.0
    per = ICP_THREADS * ICP_QB
    tiles_q = (Q + per - 1) // per
    xb = x[b]                                                    # (C, Q, 3): the nearest pred points, re-transformed
    yb = icp_transform(xb, rot[:, None], params[:, None, 9:], params[:, None, :3])
    v = _pad(contribution(xb, yb, g[None].expand(C, Q, 3)), tiles_q * per).reshape(C, tiles_q, ICP_QB, ICP_THREADS, 13)
    s_gp = _in_order(block_sum(_in_order(v.transpose(2, 3))))
    w = torch.full((13,), 2.0, dtype=torch.float64, device=x.device)
    w[0] = 1.0
    # divide by tensors: torch multiplies by the reciprocal when a CUDA tensor is divided by a Python number
    return (w * s_pg) / torch.full_like(w, P) + (w * s_gp) / torch.full_like(w, Q)


def fsum_sums(x: torch.Tensor, g: torch.Tensor, rot: torch.Tensor, params: torch.Tensor) -> torch.Tensor:
    """The same (C, 13) sums without any of the kernel's orders, for clouds and transforms on which every fp32 step is
    exact (dyadic coordinates, signed-permutation R, power-of-two s): fp64 arithmetic, fp64 nearest neighbours and
    correctly rounded `math.fsum` totals.  CPU only."""
    import math

    x, g, rot, params = x.double().cpu(), g.double().cpu(), rot.double().cpu(), params.double().cpu()
    P, Q = x.shape[0], g.shape[0]
    out = torch.zeros(rot.shape[0], 13, dtype=torch.float64)
    for n in range(rot.shape[0]):
        y = (params[n, 9:] * x) @ rot[n] + params[n, :3]
        d = ((y[:, None, :] - g[None]) ** 2).sum(-1)
        a, b = d.argmin(1), d.argmin(0)
        for k, (v1, v2) in enumerate(zip(contribution(x, y, g[a]).T, contribution(x[b], y[b], g).T)):
            w = 1.0 if k == 0 else 2.0
            out[n, k] = w * math.fsum(v1.tolist()) / P + w * math.fsum(v2.tolist()) / Q
    return out


def transform_points(p: torch.Tensor, tf: torch.Tensor) -> torch.Tensor:
    """icp.cu::icp_transform_points_kernel: p (F, N, 3), tf (F | 1, 15) = R, T, s -> (F, N, 3).  m_l = fl(s_k R[k][l]) first,
    then o_l = fl(fma(p.z, m2, fma(p.y, m1, fl(p.x m0))) + T_l)."""
    R, T, s = tf[:, None, :9].reshape(-1, 1, 3, 3), tf[:, None, 9:12], tf[:, None, 12:15]
    out = []
    for l in range(3):
        m0, m1, m2 = s[..., 0] * R[..., 0, l], s[..., 1] * R[..., 1, l], s[..., 2] * R[..., 2, l]
        out.append(fma32(p[..., 2], m2, fma32(p[..., 1], m1, p[..., 0] * m0)) + T[..., l])
    return torch.stack(out, -1)


def lattice(n: int, seed: int, dup: int = 1) -> torch.Tensor:
    """n points with coordinates k/8, |k| <= 12, each drawn point repeated about `dup` times at random indices."""
    gen = torch.Generator().manual_seed(seed)
    pts = torch.randint(-12, 13, (n // dup + 1, 3), generator=gen).float() / 8
    return pts[torch.randint(0, pts.shape[0], (n,), generator=gen)]


def lattice_transforms(C: int, seed: int):
    """Signed-permutation R, s in {1/2, 1, 2}, T in multiples of 1/8: (rot (C, 3, 3), params (C, 12)) with exact fp32
    transforms."""
    gen = torch.Generator().manual_seed(seed)
    rot = torch.zeros(C, 3, 3)
    for n in range(C):
        perm = torch.randperm(3, generator=gen)
        rot[n, torch.arange(3), perm] = torch.randint(0, 2, (3,), generator=gen).float() * 2 - 1
    params = torch.zeros(C, 12)
    params[:, :3] = torch.randint(-8, 9, (C, 3), generator=gen).float() / 8
    params[:, 9:] = torch.tensor([0.5, 1.0, 2.0])[torch.randint(0, 3, (C, 3), generator=gen)]
    return rot, params


def bits(t: torch.Tensor) -> torch.Tensor:
    """The bit pattern of a float tensor, for comparisons that tell -0 from +0 and NaN from NaN."""
    return t.view({torch.float32: torch.int32, torch.float64: torch.int64}[t.dtype])


def assert_bits_equal(got: torch.Tensor, want: torch.Tensor, what: str = "") -> None:
    got, want = got.to(want.device), want
    assert got.shape == want.shape, (what, got.shape, want.shape)
    diff = bits(got) != bits(want)
    if bool(diff.any()):
        where = diff.nonzero()[:5].tolist()
        pairs = [(float(got[tuple(w)]), float(want[tuple(w)])) for w in where]
        raise AssertionError(f"{what}: {int(diff.sum())} of {diff.numel()} differ, first at {where}: {pairs}")
