"""Flash attention on 176-key K/V tiles (-m gpu): head_dim 128 with at least 4096 keys per chunk runs on 176-key tiles,
everything else on 128-key tiles (DESIGN 4.1).  Element-by-element bounds at the tails the wider tile creates, either side
of the threshold, and the invariances of DESIGN 5 for the 176-key width.

The smallest call on the 176-key path has 24 tiles per chunk (4096 keys), so "one tile" here means a row whose keys fill
whole tiles with no tail.  Every output is a view into a NaN-filled buffer whose hidden elements must stay untouched.
"""
import math

import pytest
import torch

import kernel_exact as kx

pytestmark = pytest.mark.gpu
DEV = "cuda"
D = 128
LONG_BK = 176
LONG_MIN_KEYS = 4096


@pytest.fixture(scope="module")
def ops(amb_lib):
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from actionmesh_b200 import ops as o

    return o


def tile_width(sk_chunk: int) -> int:
    return LONG_BK if sk_chunk >= LONG_MIN_KEYS else 128


def bound_rows(q, k, v, scale, b, h, rows, sk_chunk, chunks):
    """kernel_exact.attn_bound_rows with the fp32 accumulation of o over the tile width the call runs on: its
    (2 * 128 + 4 * tiles + 40) u becomes (2 * BK + 4 * tiles + 40) u of max_k |v_kd|."""
    bk = tile_width(sk_chunk)
    tiles = chunks * ((sk_chunk + bk - 1) // bk)
    o64, bound = kx.attn_bound_rows(q, k, v, scale, b, h, rows, tiles)
    vmax = v.double().abs().amax(0, keepdim=True)
    return o64, bound + 2 * (bk - 128) * kx.U * vmax


TAIL_CASES = [
    # name, B, H, Sq, keys per chunk, kv_chunks, k scale
    ("whole_tiles_4224", 1, 2, 300, 24 * 176, 1, 1.0),           # no tail: every tile is full
    ("tail_1key_4225", 1, 2, 300, 24 * 176 + 1, 1, 0.25),        # the last tile holds one key
    ("tail_16k_4256", 1, 2, 300, 24 * 176 + 32, 1, 0.25),        # a tail of whole 16-key P·V steps
    ("window_32784_tail48", 1, 2, 300, 32784, 1, 1.0),           # the default window: 186 tiles + 48 keys
    ("chunks8_4098", 1, 2, 300, 4098, 8, 0.25),                  # ragged chunks: a 50-key tail in each
    ("below_threshold_4095", 2, 2, 300, 4095, 1, 0.25),          # 128-key tiles (31 + a 127-key tail)
    ("at_threshold_4096", 2, 2, 300, 4096, 1, 0.25),             # 176-key tiles (23 + a 48-key tail)
]


@pytest.mark.parametrize("name,B,H,Sq,skc,chunks,kscale", TAIL_CASES, ids=[c[0] for c in TAIL_CASES])
def test_tile_tails_elementwise(ops, name, B, H, Sq, skc, chunks, kscale):
    """Sampled rows of every (batch, head) within the bound; v is U[0.5, 1.5) so a lost or extra key shifts the row."""
    Sk = skc * chunks
    g = torch.Generator(device=DEV).manual_seed(17)
    q = kx.attn_tensor(B, Sq, H, D, g, DEV)
    k = kx.attn_tensor(B, Sk, H, D, g, DEV, chunks=chunks, scale=kscale)
    v = kx.attn_tensor(B, Sk, H, D, g, DEV, chunks=chunks, kind="uniform")
    obuf, o = kx.attn_out(B, Sq, H, D, DEV)
    scale = 1.0 / math.sqrt(D)
    ops.flash_attn(q, k, v, o, scale, kv_chunks=chunks)
    assert bool(torch.isfinite(o).all()), f"{name}: non-finite output"
    rows = kx.sample_rows(Sq, torch.Generator().manual_seed(1)).to(DEV)
    for b in range(B):
        for h in range(H):
            kb = k[b, ..., h, :].reshape(Sk, D)
            vb = v[b, ..., h, :].reshape(Sk, D)
            o64, bound = bound_rows(q, kb, vb, scale, b, h, rows, skc, chunks)
            kx.compare(o[b, rows, h], o64, bound, f"{name} b={b} h={h}", store_rounding=False)
    kx.int_view(o).fill_(kx.NAN_BF16)
    assert kx.is_untouched(obuf), f"{name}: wrote outside the output view"


def _qkv(B, Sq, Sk, H, seed=3):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (kx.attn_tensor(B, Sq, H, D, g, DEV), kx.attn_tensor(B, Sk, H, D, g, DEV),
            kx.attn_tensor(B, Sk, H, D, g, DEV, kind="uniform"))


@pytest.mark.parametrize("tiles_per_chunk", [24, 25])
def test_whole_176_tile_chunks_are_bit_exact(ops, tiles_per_chunk):
    """kv_chunks of whole 176-key tiles visit the same tiles in the same order as one call over all keys.  24 tiles
    (4224 keys) are also 33 whole 128-key tiles; 25 tiles (4400 keys) are not, so this case holds only if both calls
    run on 176-key tiles."""
    skc = tiles_per_chunk * LONG_BK
    q, k, v = _qkv(2, 300, 4 * skc, 2)
    _, o = kx.attn_out(2, 300, 2, D, DEV)
    ops.flash_attn(q, k, v, o, 1 / math.sqrt(D))
    k5, v5 = k.unflatten(1, (4, skc)), v.unflatten(1, (4, skc))
    obuf, oc = kx.attn_out(2, 300, 2, D, DEV)
    ops.flash_attn(q, k5, v5, oc, 1 / math.sqrt(D), kv_chunks=4)
    assert torch.equal(kx.int_view(oc), kx.int_view(o))
    kx.int_view(oc).fill_(kx.NAN_BF16)
    assert kx.is_untouched(obuf)


def test_query_slice_is_bit_exact_176(ops):
    """Rows are independent on the 176-key path: the call on query rows [37, Sq) equals those rows of the full call."""
    q, k, v = _qkv(2, 700, 5000, 3)
    _, o = kx.attn_out(2, 700, 3, D, DEV)
    ops.flash_attn(q, k, v, o, 1 / math.sqrt(D))
    obuf, os_ = kx.attn_out(2, 700 - 37, 3, D, DEV)
    ops.flash_attn(q[:, 37:], k, v, os_, 1 / math.sqrt(D))
    assert torch.equal(kx.int_view(os_), kx.int_view(o[:, 37:]))
    kx.int_view(os_).fill_(kx.NAN_BF16)
    assert kx.is_untouched(obuf)


def test_single_head_is_bit_exact_176(ops):
    """One (batch, head) call on the 176-key path equals its slice of the full call bit for bit."""
    q, k, v = _qkv(2, 300, 4500, 4)
    _, o = kx.attn_out(2, 300, 4, D, DEV)
    ops.flash_attn(q, k, v, o, 1 / math.sqrt(D))
    _, o1 = kx.attn_out(1, 300, 1, D, DEV)
    ops.flash_attn(q[1:2, :, 3:4], k[1:2, :, 3:4], v[1:2, :, 3:4], o1, 1 / math.sqrt(D))
    assert torch.equal(kx.int_view(o1), kx.int_view(o[1:2, :, 3:4]))
