"""Element-by-element checks of the GEMM and flash-attention kernels (-m gpu) against exact or bounded fp64 results.

GEMM: operands on the dyadic grids of tests/kernel_exact.py, so the linear epilogues must be bit-exact and GELU / RMSNorm
/ RoPE must meet the per-element bounds derived there.  Every epilogue configuration the library launches (GEMM_CONFIGS)
runs at small and odd M values, and the DiT's block GEMMs, one TripoSG-decoder GEMM and one DinoV2-L GEMM run at their
production sizes.  Flash attention: a per-element bound on sampled rows (kernel_exact.attn_bound_rows) at the pipeline's
shapes, and invariances that must hold bit for bit.  Every output is a view into a NaN-filled buffer whose hidden elements
must stay untouched, and every operand hides NaN past its last column.
"""
import math

import pytest
import torch

import kernel_exact as kx

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def ops(amb_lib):
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from actionmesh_b200 import ops as o

    return o


@pytest.fixture
def exact_torch_matmul():
    """fp32 matmuls without TF32 and bf16 matmuls without reduced-precision reductions, restored afterwards."""
    saved = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cuda.matmul.allow_bf16_reduced_precision_reduction)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cuda.matmul.allow_bf16_reduced_precision_reduction = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cuda.matmul.allow_bf16_reduced_precision_reduction = saved


def test_cublas_reproduces_the_exact_grid(exact_torch_matmul):
    """The premise of the exact GEMM checks, tested on a library that is not ours: on the grids at K = 8192, cuBLAS's fp32
    GEMM equals the fp64 result bit for bit, and its bf16 GEMM equals the fp64 result rounded to bf16."""
    g = torch.Generator(device=DEV).manual_seed(11)
    a = kx.grid((1024, 8192), 8, 8, g, DEV)
    w = kx.grid((512, 8192), 8, 16, g, DEV)
    exact = a.double() @ w.double().t()
    assert torch.equal(exact.float().double(), exact)
    assert torch.equal(kx.int_view(a.float() @ w.float().t()), kx.int_view(exact.float()))
    assert torch.equal(kx.int_view(a @ w.t()), kx.int_view(exact.bfloat16()))


@pytest.mark.parametrize("name", [c.name for c in kx.GEMM_CONFIGS])
def test_gemm_config_table(ops, name):
    """One configuration at every M of SMALL_MS with padded operands and outputs, and at m = 129 exactly sized."""
    cfg = kx.GEMM_CONFIG[name]
    for i, m in enumerate(kx.SMALL_MS):
        case = kx.build_gemm_case(cfg, m, DEV, seed=i)
        case.call(ops.gemm)
        kx.check_gemm(case)
    case = kx.build_gemm_case(cfg, 129, DEV, seed=99, pad=False)
    case.call(ops.gemm)
    kx.check_gemm(case)


PRODUCTION = [
    # the DiT at the default window (M = 2 CFG branches x 16 frames x 2049 tokens): the six block GEMMs
    (65568, kx.GemmConfig("dit_attn_out_res_f32", 2048, 2048, out="f32", bias=True, residual="alias", res="f32")),
    (65568, kx.GemmConfig("dit_qkv_norm_rope", 6144, 2048, norm="qkv_rope", rows_per_pos=2049)),
    (65568, kx.GemmConfig("dit_ff1_gelu", 8192, 2048, bias=True, act=1)),
    (65568, kx.GemmConfig("dit_ff2_res_out2", 2048, 8192, out="f32", bias=True, residual="alias", res="f32", out2=True)),
    (65568, kx.GemmConfig("dit_skip_a2", 2048, 4096, bias=True, k_split=2048)),
    # one 262 144-row query chunk of the TripoSG decoder, and DinoV2-L's LayerScale MLP output over 16 frames
    (262144, kx.GemmConfig("triposg_query_ff1_gelu", 4096, 1024, bias=True, act=1)),
    (16 * 257, kx.GemmConfig("dinov2l_fc2_ls_res_f32", 1024, 4096, out="f32", bias=True, col_scale=True, residual="alias",
                             res="f32")),
]


@pytest.mark.parametrize("m,cfg", PRODUCTION, ids=[c.name for _, c in PRODUCTION])
def test_gemm_production_shapes(ops, m, cfg):
    """Every element at the sizes the persistent schedule runs: band rasterisation over 257 M-tile pairs, and the ring
    phase wrapping over 128 k-blocks at K = 8192."""
    case = kx.build_gemm_case(cfg, m, DEV, seed=5)
    case.call(ops.gemm)
    kx.check_gemm(case)
    del case
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------- attention
ATTN_CASES = [
    # name, B, H, Sq, Sk, D, kv_chunks, k scale (small logits make a masked key that slips in visible)
    ("self_window_32784", 2, 16, 32784, 32784, 128, 1, 1.0),
    ("cross_2049x257", 16, 16, 2049, 257, 128, 1, 0.25),
    ("triposg_query_262144x2048", 1, 8, 262144, 2048, 128, 1, 1.0),
    ("d64_2048x2048", 1, 8, 2048, 2048, 64, 1, 1.0),
    ("d64_2048x16384", 1, 8, 2048, 16384, 64, 1, 1.0),
    ("d64_chunks4_200keys", 2, 2, 300, 800, 64, 4, 0.25),
    ("d128_chunks8_64keys", 1, 2, 64, 512, 128, 8, 0.25),
    ("d128_chunks4_200keys", 2, 2, 300, 800, 128, 4, 0.25),
    ("d128_q129_k129", 1, 3, 129, 129, 128, 1, 0.25),
]


@pytest.mark.parametrize("name,B,H,Sq,Sk,D,chunks,kscale", ATTN_CASES, ids=[c[0] for c in ATTN_CASES])
def test_flash_attention_elementwise(ops, name, B, H, Sq, Sk, D, chunks, kscale):
    """Sampled rows of every (batch, head) within the bound of kernel_exact.attn_bound_rows; v is U[0.5, 1.5) so the
    output is O(1) and a lost or extra key shows as a shift of the whole row."""
    g = torch.Generator(device=DEV).manual_seed(7)
    q = kx.attn_tensor(B, Sq, H, D, g, DEV)
    k = kx.attn_tensor(B, Sk, H, D, g, DEV, chunks=chunks, scale=kscale)
    v = kx.attn_tensor(B, Sk, H, D, g, DEV, chunks=chunks, kind="uniform")
    obuf, o = kx.attn_out(B, Sq, H, D, DEV)
    scale = 1.0 / math.sqrt(D)
    ops.flash_attn(q, k, v, o, scale, kv_chunks=chunks)
    assert bool(torch.isfinite(o).all()), f"{name}: non-finite output"
    rows = kx.sample_rows(Sq, torch.Generator().manual_seed(1)).to(DEV)
    tiles = chunks * ((Sk // chunks + 127) // 128)
    for b in range(B):
        for h in range(H):
            kb = k[b, ..., h, :].reshape(Sk, D)
            vb = v[b, ..., h, :].reshape(Sk, D)
            o64, bound = kx.attn_bound_rows(q, kb, vb, scale, b, h, rows, tiles)
            kx.compare(o[b, rows, h], o64, bound, f"{name} b={b} h={h}", store_rounding=False)
    kx.int_view(o).fill_(kx.NAN_BF16)
    assert kx.is_untouched(obuf), f"{name}: wrote outside the output view"


def _qkv(B, Sq, Sk, H, D, seed=3):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (kx.attn_tensor(B, Sq, H, D, g, DEV), kx.attn_tensor(B, Sk, H, D, g, DEV),
            kx.attn_tensor(B, Sk, H, D, g, DEV, kind="uniform"))


@pytest.mark.parametrize("D", [128, 64])
def test_attention_query_slice_is_bit_exact(ops, D):
    """Rows are independent: the call on query rows [37, Sq) equals those rows of the full call bit for bit."""
    q, k, v = _qkv(2, 700, 1000, 3, D)
    _, o = kx.attn_out(2, 700, 3, D, DEV)
    ops.flash_attn(q, k, v, o, 1 / math.sqrt(D))
    obuf, os_ = kx.attn_out(2, 700 - 37, 3, D, DEV)
    ops.flash_attn(q[:, 37:], k, v, os_, 1 / math.sqrt(D))
    assert torch.equal(kx.int_view(os_), kx.int_view(o[:, 37:]))
    kx.int_view(os_).fill_(kx.NAN_BF16)
    assert kx.is_untouched(obuf)


@pytest.mark.parametrize("D", [128, 64])
def test_attention_single_head_is_bit_exact(ops, D):
    """One (batch, head) call equals its slice of the full call bit for bit."""
    q, k, v = _qkv(2, 300, 257, 4, D)
    _, o = kx.attn_out(2, 300, 4, D, DEV)
    ops.flash_attn(q, k, v, o, 1 / math.sqrt(D))
    _, o1 = kx.attn_out(1, 300, 1, D, DEV)
    ops.flash_attn(q[1:2, :, 3:4], k[1:2, :, 3:4], v[1:2, :, 3:4], o1, 1 / math.sqrt(D))
    assert torch.equal(kx.int_view(o1), kx.int_view(o[1:2, :, 3:4]))


@pytest.mark.parametrize("D", [128, 64])
def test_attention_whole_tile_chunks_are_bit_exact(ops, D):
    """kv_chunks whose chunks are whole 128-key tiles visit the same tiles in the same order as one call (DESIGN 5)."""
    q, k, v = _qkv(2, 300, 4 * 256, 2, D)
    _, o = kx.attn_out(2, 300, 2, D, DEV)
    ops.flash_attn(q, k, v, o, 1 / math.sqrt(D))
    k5, v5 = k.unflatten(1, (4, 256)), v.unflatten(1, (4, 256))
    _, oc = kx.attn_out(2, 300, 2, D, DEV)
    ops.flash_attn(q, k5, v5, oc, 1 / math.sqrt(D), kv_chunks=4)
    assert torch.equal(kx.int_view(oc), kx.int_view(o))
