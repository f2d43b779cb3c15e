"""The premises of tests/icp_exact.py, on the host: fma32 is libm's fmaf bit for bit (and plain fp64 is not), the block
sum is lane 0 of a scalar simulation of __shfl_down_sync, and on dyadic lattices every restated fp32 step is exact, so
the kernel's sums there equal an order-free exact sum.  The GPU side is tests/test_icp_exact_gpu.py."""
from __future__ import annotations

import ctypes
import ctypes.util
import math
import random

import pytest
import torch

import icp_exact as ex
import icp_ref as ref


@pytest.fixture(scope="module")
def fmaf():
    libm = ctypes.CDLL(ctypes.util.find_library("m"))
    libm.fmaf.restype = ctypes.c_float
    libm.fmaf.argtypes = [ctypes.c_float] * 3
    return lambda a, b, c: torch.tensor([libm.fmaf(x, y, z) for x, y, z in zip(a.tolist(), b.tolist(), c.tolist())])


def _midpoint_triples():
    """(1 + i 2^-12)(1 + j 2^-12) with i, j odd is exactly halfway between two fp32 numbers; c = 0 leaves the
    tie to even and a tiny c of either sign decides it.  Scaled by powers of two for other exponents."""
    a, b, c = [], [], []
    for i in range(1, 64, 2):
        for j in range(1, 64, 6):
            for t in (0.0, 2.0 ** -60, -2.0 ** -60, 2.0 ** -75, -2.0 ** -70):
                for e in (0, -20, 37):
                    a.append((1 + i * 2.0 ** -12) * 2.0 ** e)
                    b.append(1 + j * 2.0 ** -12)
                    c.append(t * 2.0 ** e)
    return torch.tensor(a), torch.tensor(b), torch.tensor(c)


def test_fma32_is_fmaf(fmaf):
    gen = torch.Generator().manual_seed(0)
    n = 50_000
    a = torch.randn(n, generator=gen) * torch.exp2(torch.randint(-30, 30, (n,), generator=gen).float())
    b = torch.randn(n, generator=gen) * torch.exp2(torch.randint(-30, 30, (n,), generator=gen).float())
    c = (a * b) * torch.randn(n, generator=gen) * torch.exp2(torch.randint(-26, 4, (n,), generator=gen).float())
    ex.assert_bits_equal(ex.fma32(a, b, c), fmaf(a, b, c), "random")
    ex.assert_bits_equal(ex.fma32(a, b, -(a * b)), fmaf(a, b, -(a * b)), "cancellation")   # the product's rounding error
    assert bool((ex.fma32(a, b, -(a * b)) != 0).any())
    ma, mb, mc = _midpoint_triples()
    ex.assert_bits_equal(ex.fma32(ma, mb, mc), fmaf(ma, mb, mc), "midpoints")
    one = torch.tensor([1 + 2.0 ** -12])
    tiny = torch.tensor([2.0 ** -60])
    assert int(ex.bits(ex.fma32(one, one, tiny))) == 0x3F801001
    assert int(ex.bits(ex.naive_fma32(one, one, tiny))) == 0x3F801000                     # fp64 double-rounds
    assert bool((ex.bits(ex.naive_fma32(ma, mb, mc)) != ex.bits(fmaf(ma, mb, mc))).any())


def _shfl_down_lane0(vals: list[float]) -> float:
    """32 lanes of `a += __shfl_down_sync(~0, a, o)`: a lane whose source lane l + o is past 31 reads its own value."""
    a = list(vals)
    for o in (16, 8, 4, 2, 1):
        a = [a[l] + (a[l + o] if l + o < 32 else a[l]) for l in range(32)]
    return a[0]


def test_block_sum_is_the_shuffle_tree():
    rng = random.Random(1)
    for _ in range(50):
        v = [rng.choice((1, -1)) * rng.random() * 2.0 ** rng.randint(-40, 40) for _ in range(ex.ICP_THREADS)]
        warps = [_shfl_down_lane0(v[32 * w:32 * w + 32]) for w in range(ex.ICP_THREADS // 32)]
        want = 0.0
        for w in warps:
            want += w
        t = torch.tensor(v, dtype=torch.float64)
        assert float(ex.warp_tree(t[:32, None])[0]) == warps[0]
        assert float(ex.block_sum(t[:, None])[0]) == want


def test_block_sum_order_matters():
    """The tree is not interchangeable with other orders: on mixed-sign values it differs from a sequential sum, and from
    the exact sum, in about half the trials."""
    rng = random.Random(2)
    trials = [[rng.choice((1, -1)) * rng.random() * 2.0 ** rng.randint(-8, 8) for _ in range(ex.ICP_THREADS)]
              for _ in range(50)]
    tree = [float(ex.block_sum(torch.tensor(v, dtype=torch.float64)[:, None])[0]) for v in trials]
    assert sum(t != sum(v) for t, v in zip(tree, trials)) >= 20
    assert sum(t != math.fsum(v) for t, v in zip(tree, trials)) >= 20


def test_lattice_steps_are_exact():
    x, g = ex.lattice(300, 3), ex.lattice(250, 4)
    rot, params = ex.lattice_transforms(6, 5)
    y = ex.icp_transform(x[None], rot[:, None], params[:, None, 9:], params[:, None, :3])
    y64 = torch.stack([(params[n, 9:].double() * x.double()) @ rot[n].double() + params[n, :3].double() for n in range(6)])
    assert torch.equal(y.double(), y64)
    d = ex.dist2(y[:, :, None], g[None, None])
    assert torch.equal(d.double(), ((y64[:, :, None] - g.double()[None, None]) ** 2).sum(-1))
    tf = torch.cat([rot.reshape(6, 9), params[:, :3], params[:, 9:]], 1)
    assert torch.equal(ex.transform_points(x[None].expand(6, -1, -1), tf).double(), y64)


@pytest.mark.parametrize("P,Q,C", [(300, 250, 3), (1025, 700, 2), (129, 1030, 9)])
def test_lattice_sums_equal_the_exact_sums(P, Q, C):
    """On the lattice the kernel's order gives the exact sums, so the restatement must equal an order-free fsum."""
    x, g = ex.lattice(P, P, dup=4), ex.lattice(Q, Q, dup=4)
    rot, params = ex.lattice_transforms(C, C)
    ex.assert_bits_equal(ex.icp_sums(x, g, rot, params), ex.fsum_sums(x, g, rot, params), "lattice sums")


def test_sums_agree_with_icp_ref():
    """The restatement's layout (x ⊗ e index order, scales, which point pairs with which) agrees with icp_ref.chamfer_sums
    on the same nearest-neighbour choices, to the fp32 rounding of y (|y| ~ 1, so about 1e-7 against sums of order 0.1)."""
    gen = torch.Generator().manual_seed(6)
    x, g = torch.randn(700, 3, generator=gen), torch.randn(650, 3, generator=gen)
    params = ref.initial_state(5) + 0.05 * torch.randn(5, 12, generator=gen)
    rot = ref.rot6d_to_matrix(params[:, 3:9])
    got = ex.icp_sums(x, g, rot, params)
    _, a, b = ex.icp_nearest(x, g, rot, params)
    want = ref.chamfer_sums(x.double(), g.double(), rot.double(), params[:, 9:].double(), params[:, :3].double(), a=a, b=b)
    assert float((got - want).abs().max()) <= 1e-6


def test_nearest_takes_the_first_minimum():
    q = torch.tensor([[0.0, 0.0, 0.0], [1.0, 1.0, 1.0]])
    r = torch.tensor([[2.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, -1.0], [1.0, 1.0, 1.0], [1.0, 1.0, 1.0]])
    d, i = ex.nearest(q, r)
    assert i.tolist() == [1, 3] and d.tolist() == [1.0, 0.0]
