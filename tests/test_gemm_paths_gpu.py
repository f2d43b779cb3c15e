"""The GEMM's cooperative 128 x 256 path (-m gpu), element by element on the exact grids of tests/kernel_exact.py.

amb_gemm_bf16 runs 128 x 256 tiles with cooperative consumers when N is a multiple of 256 and K > 2048; otherwise 128 x 128
tiles with ping-pong consumers (or 128 x 64 when N is not a multiple of 128).  The configuration table of kernel_exact runs
at K <= 256, so test_kernel_exactness_gpu checks every epilogue on ping-pong; here every epilogue runs again at K = 4096,
on the cooperative path.  The two paths must also agree bit for bit: each output element sums its k16 steps in the same
order into one fp32 accumulator on both.
"""
import dataclasses

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


def coop_config(cfg: kx.GemmConfig, k: int = 4096) -> kx.GemmConfig:
    """The configuration at K = 4096 and N rounded up to a multiple of 256 (768 for the layouts in thirds).  The A split
    stays after the first k-block, in the middle, or before the last k-block."""
    n = cfg.n if cfg.n % 256 == 0 else (768 if cfg.norm in ("qkv", "qkv_rope", "rope") else 256 * (cfg.n // 256 + 1))
    ks = cfg.k_split
    if ks is not None:
        ks = 64 if ks == 64 else (k - 64 if ks == cfg.k - 64 else k * ks // cfg.k)
    return dataclasses.replace(cfg, name=cfg.name + "_coop", n=n, k=k, k_split=ks)


@pytest.mark.parametrize("name", [c.name for c in kx.GEMM_CONFIGS])
def test_cooperative_path(ops, name):
    """Every M of SMALL_MS (one row, tile edges, an odd M-tile count, several tiles per cluster)."""
    cfg = coop_config(kx.GEMM_CONFIG[name])
    for i, m in enumerate(kx.SMALL_MS):
        case = kx.build_gemm_case(cfg, m, DEV, seed=i)
        case.call(ops.gemm)
        kx.check_gemm(case)


@pytest.mark.parametrize("m,k", [(1, 2112), (161 * 128 - 45, 4096), (3 * 128 + 5, 8192)])
def test_paths_agree_bit_for_bit(ops, m, k):
    """One A against a W of N = 384 (ping-pong) and against its first 256 rows (cooperative): the shared columns of the
    fp32 outputs are equal bit for bit.  Normal operands, so a different summation order would show."""
    g = torch.Generator(device=DEV).manual_seed(k + m)
    a = torch.randn(m, k, generator=g, device=DEV).bfloat16()
    w = torch.randn(384, k, generator=g, device=DEV).bfloat16()
    out384 = torch.empty(m, 384, device=DEV)
    out256 = torch.empty(m, 256, device=DEV)
    ops.gemm(a, w, out384)
    ops.gemm(a, w[:256], out256)
    assert torch.equal(kx.int_view(out384[:, :256]), kx.int_view(out256))
