"""ops refuses a tensor of the wrong device or dtype in Python, before any launch, for the tensors every wrapper hands to
the C ABI: GEMM outputs, residuals and norm/RoPE tables included."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _refused(call, name):
    from actionmesh_b200 import AmbError, ops

    before = ops.launch_count
    with pytest.raises(AmbError, match=f"^{name}: expected"):
        call()
    assert ops.launch_count == before


def test_gemm_refuses_bad_out_residual_and_tables(amb_lib):
    from actionmesh_b200 import ops

    dev = torch.device("cuda")
    a = torch.zeros(128, 128, dtype=torch.bfloat16, device=dev)
    w = torch.zeros(128, 128, dtype=torch.bfloat16, device=dev)
    out = torch.zeros(128, 128, dtype=torch.bfloat16, device=dev)
    _refused(lambda: ops.gemm(a, w, out.cpu()), "out")
    _refused(lambda: ops.gemm(a, w, out, residual=out.half()), "residual")
    cos = torch.ones(128, 64, device=dev)
    rope = dict(rope_cols=128, cos=cos.cpu(), sin=cos)
    _refused(lambda: ops.gemm(a, w, out, norm=rope), "rope cos")
    ops.gemm(a, w, out, residual=out)  # the same calls with valid tensors run
    ops.gemm(a, w, out, norm=dict(rope_cols=128, cos=cos, sin=cos))
    torch.cuda.synchronize()


def test_layernorm_refuses_cpu_input(amb_lib):
    from actionmesh_b200 import ops

    dev = torch.device("cuda")
    x = torch.zeros(4, 256, dtype=torch.bfloat16)
    gamma, beta = torch.ones(256, device=dev), torch.zeros(256, device=dev)
    out = torch.empty(4, 256, dtype=torch.bfloat16, device=dev)
    _refused(lambda: ops.layernorm(x, gamma, beta, 1e-5, out=out), "x")
    ops.layernorm(x.to(dev), gamma, beta, 1e-5, out=out)
    torch.cuda.synchronize()
