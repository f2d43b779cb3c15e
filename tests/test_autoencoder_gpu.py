"""Stage-II parity (-m gpu): B200Autoencoder (CUDA, through the C ABI) against
  (1) the golden displacement field produced by the reference's own ActionMeshAutoencoder (tests/golden/autoencoder_tiny.pt),
  (2) the fp32 oracle restatement with the trunk removed (num_layers=0): isolates the vertex-query path, which the
      reference runs in fp32 (temporal_autoencoder.py:264-266) and this library evaluates with split-bf16 operands ->
      fp32-grade tolerance,
  (3) the oracle at full width (1024, 8 heads) with a short trunk, also reporting the ActionBench Chamfer distance between
      the two vertex sets.
Stated tolerances: trunk = bf16 GEMM operands with fp32 accumulation and fp32 residual stream (the reference's own CUDA
recipe) vs the fp32 CPU oracle -> |d displacement| < 2e-2; query path alone -> < 5e-5."""
import json
import os
import tempfile

import pytest
import torch

from conftest import load_golden
from oracle import autoencoder_oracle as ao

REPORT_DIR = os.path.join(tempfile.gettempdir(), "actionmesh_b200_reports")

pytestmark = pytest.mark.gpu


def _model(cfg: "ao.AutoencoderConfig", sd):
    from actionmesh_b200.autoencoder import AutoencoderConfig, B200Autoencoder

    m = B200Autoencoder(AutoencoderConfig(width=cfg.width, num_layers=cfg.num_layers,
                                          num_attention_heads=cfg.num_attention_heads)).to("cuda")
    m.load_state_dict(sd)
    return m


def test_split3_and_softmax_kernels(amb_lib):
    from actionmesh_b200 import ops

    g = torch.Generator().manual_seed(3)
    x = (torch.randn(37, 256, generator=g) * 3).cuda()
    a = ops.split3(x, torch.empty(37, 768, dtype=torch.bfloat16, device="cuda"), seg=128).float()
    w = ops.split3(x, torch.empty(37, 768, dtype=torch.bfloat16, device="cuda"), seg=128, weight=True).float()
    for s in range(2):
        hi, lo = a[:, s * 384:s * 384 + 128], a[:, s * 384 + 128:s * 384 + 256]
        assert torch.equal(hi, a[:, s * 384 + 256:s * 384 + 384])
        assert torch.equal(hi, x[:, s * 128:(s + 1) * 128].bfloat16().float())
        assert ((hi + lo) - x[:, s * 128:(s + 1) * 128]).abs().max() <= 2 ** -16 * x.abs().max()
        assert torch.equal(w[:, s * 384:s * 384 + 128], hi) and torch.equal(w[:, s * 384 + 128:s * 384 + 256], hi)
        assert torch.equal(w[:, s * 384 + 256:s * 384 + 384], lo)
    # split GEMM == fp32 matmul to ~1e-5 relative
    from actionmesh_b200 import ops as o
    A = torch.randn(300, 192, generator=g).cuda()
    W = torch.randn(128, 192, generator=g).cuda()
    a3 = o.split3(A, torch.empty(300, 576, dtype=torch.bfloat16, device="cuda"))
    w3 = o.split3(W, torch.empty(128, 576, dtype=torch.bfloat16, device="cuda"), weight=True)
    c = o.gemm(a3, w3, torch.empty(300, 128, dtype=torch.float32, device="cuda"))
    ref = (A.double() @ W.double().t()).float()
    assert (c - ref).abs().max() < 2e-4 * ref.abs().max()
    # softmax
    s = (torch.randn(5, 128, generator=g) * 4).cuda()
    p3 = o.softmax_split3(s, 100, 0.5, torch.empty(5, 384, dtype=torch.bfloat16, device="cuda")).float()
    p = torch.softmax(s[:, :100] * 0.5, dim=-1)
    assert ((p3[:, :100] + p3[:, 128:228]) - p).abs().max() < 1e-6
    assert torch.equal(p3[:, :128], p3[:, 256:384]) and p3[:, 100:128].abs().max() == 0 and p3[:, 228:256].abs().max() == 0


def test_matches_reference_module_golden(amb_lib):
    g = load_golden("autoencoder_tiny.pt")
    cfg = ao.AutoencoderConfig(**g["config"])
    m = _model(cfg, ao.make_autoencoder_state_dict(cfg, g["seed"]))
    out = m.forward(g["latent"], g["framestep"], g["source_alpha"], g["target_alphas"], g["query"]).cpu()
    ref = g["displacement"]
    assert out.shape == ref.shape
    err = (out - ref).abs().max().item()
    assert err < 2e-2, err


def test_query_path_is_fp32_grade(amb_lib):
    cfg = ao.AutoencoderConfig(width=256, num_layers=0, num_attention_heads=2)
    sd = ao.make_autoencoder_state_dict(cfg, 77)
    gen = torch.Generator().manual_seed(5)
    lat = torch.randn(1, 3, 30, 64, generator=gen).bfloat16().float()  # bf16-representable: post_quant is then exact
    fs = torch.tensor([[5.0, 6.0, 9.0]])  # R = 3 * 31 = 93 keys: odd, exercises the padded / masked softmax tail
    sa, ta = torch.tensor([0.25]), torch.tensor([[0.0, 0.6]])
    q = torch.rand(1, 700, 6, generator=gen) * 2 - 1
    m = _model(cfg, sd)
    out = m.forward(lat, fs, sa, ta, q).cpu()
    ref = ao.autoencoder_forward(sd, cfg, lat, fs, sa, ta, q)
    err = (out - ref).abs().max().item()
    assert err < 5e-5, err


def test_full_width_vs_oracle_with_chamfer(amb_lib):
    cfg = ao.AutoencoderConfig(width=1024, num_layers=2, num_attention_heads=8)
    sd = ao.make_autoencoder_state_dict(cfg, 4321)
    gen = torch.Generator().manual_seed(9)
    lat = torch.randn(1, 4, 255, 64, generator=gen)
    fs = torch.tensor([[0.0, 1.0, 2.0, 3.0]])
    sa, ta = torch.tensor([0.0]), torch.tensor([[0.0, 1.0]])
    pts = torch.randn(1, 3000, 3, generator=gen)
    pts = pts / pts.norm(dim=-1, keepdim=True) * 0.6
    q = torch.cat([pts, pts / 0.6], dim=-1)
    m = _model(cfg, sd)
    m.QUERY_CHUNK = 2048  # exercise the query chunking
    out = m.forward(lat, fs, sa, ta, q)
    v = m.apply_displacement(pts.cuda(), out).cpu()
    ref = ao.autoencoder_forward(sd, cfg, lat, fs, sa, ta, q)
    v_ref = ao.apply_displacement(pts, ref)
    err = (out.cpu() - ref).abs().max().item()
    cds = [ao.chamfer_score(v[0, t].numpy(), v_ref[0, t].numpy(), n=10_000, seed=44) for t in range(2)]
    report = {"stage2_max_abs_err": err, "stage2_chamfer": cds}
    os.makedirs(REPORT_DIR, exist_ok=True)
    json.dump(report, open(os.path.join(REPORT_DIR, "stage2_report.json"), "w"), indent=1)
    print("STAGE2", json.dumps(report))
    assert err < 2e-2, report
