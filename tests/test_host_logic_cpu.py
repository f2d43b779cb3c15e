"""Host-side mirror of the reference interfaces (no GPU): schedule, CFG, weight re-packing, windows."""
import torch

import os

from conftest import ROOT, load_golden
from actionmesh_b200.blocks import repack_cross_kv, repack_self_qkv
from actionmesh_b200.guidance import ClassifierFreeGuidance
from actionmesh_b200.scheduler import B200SchedulerFlow


def test_schedule_matches_reference_known_answers():
    host = load_golden("host_logic.pt")
    for n, (ts, ds) in host["schedule"].items():
        s = B200SchedulerFlow(num_inference_steps=n, shift=3.0)
        a, b = s.get_schedule()
        assert torch.equal(a, ts) and torch.equal(b, ds)


def test_get_noise_stream_matches_reference():
    host = load_golden("host_logic.pt")
    g = torch.Generator().manual_seed(44)
    n = B200SchedulerFlow(num_inference_steps=4).get_noise([2048, 64], 1, 16, "cpu", g)
    assert n.shape == (1, 16, 2048, 64)
    assert torch.equal(n[0, :2, :4, :8], host["noise_seed44_head"])


def test_cfg_surface():
    host = load_golden("host_logic.pt")
    cf = ClassifierFreeGuidance(guidance_at_inference=[[0, 1], [1, 1]], guidance_scales=[7.5])
    assert torch.allclose(cf.aggregate_cfg(host["cfg_in"].clone()), host["cfg_out"], atol=1e-5)
    lat, ctx = torch.randn(1, 3, 4, 8), torch.randn(1, 3, 5, 6)
    mask, fs = torch.tensor([[1.0, 0, 0]]), torch.tensor([[0.0, 1, 2]])
    l2, c2, m2, f2 = cf.cfg_at_inference(lat, ctx, mask, fs)
    assert l2.shape[0] == 2 and torch.equal(c2[0], torch.zeros_like(ctx[0])) and torch.equal(c2[1], ctx[0])
    assert torch.equal(m2[0], m2[1]) and torch.equal(f2[0], f2[1])
    assert torch.equal(cf.get_unobserved_mask(mask), mask == 0)
    assert cf.branches() == [(0, 1), (1, 1)]
    off = ClassifierFreeGuidance(inference_enabled=False)
    assert off.branches() == [(1, 1)] and off.aggregate_cfg(lat) is lat


def test_qkv_repack_equals_head_interleaved_split():
    """SURVEY A.2: permuting the rows of cat(Wq,Wk,Wv) once == the reference's split of cat(q,k,v) per head."""
    torch.manual_seed(0)
    H, dh, D = 4, 8, 32
    wq, wk, wv = torch.randn(D, D), torch.randn(D, D), torch.randn(D, D)
    x = torch.randn(5, D)
    qkv = torch.cat([x @ wq.t(), x @ wk.t(), x @ wv.t()], -1).view(5, H, 3 * dh)
    q_ref, k_ref, v_ref = qkv.split(dh, dim=-1)  # attention_processor.py:106-110
    packed = x @ repack_self_qkv(wq, wk, wv, H).t()
    q, k, v = packed[:, :D].view(5, H, dh), packed[:, D:2 * D].view(5, H, dh), packed[:, 2 * D:].view(5, H, dh)
    assert torch.allclose(q, q_ref, atol=1e-5) and torch.allclose(k, k_ref, atol=1e-5) and torch.allclose(v, v_ref, atol=1e-5)
    Dc = 16
    wk2, wv2 = torch.randn(D, Dc), torch.randn(D, Dc)
    c = torch.randn(7, Dc)
    kv = torch.cat([c @ wk2.t(), c @ wv2.t()], -1).view(7, H, 2 * dh)
    k_ref, v_ref = kv.split(dh, dim=-1)  # :111-115
    packed = c @ repack_cross_kv(wk2, wv2, H).t()
    assert torch.allclose(packed[:, :D].view(7, H, dh), k_ref, atol=1e-5)
    assert torch.allclose(packed[:, D:].view(7, H, dh), v_ref, atol=1e-5)


def test_windows_and_bank_match_reference_known_answers():
    from actionmesh_b200.windows import LatentBank, chunk_from

    host = load_golden("host_logic.pt")
    for args, ref in host["chunk_from"].items():
        got = chunk_from(*args)
        assert len(got) == len(ref) and all(torch.equal(a, b) for a, b in zip(got, ref)), args
    bank = LatentBank(empty_dims=(4, 2))
    bank.update(torch.tensor([3.0]), torch.ones(1, 4, 2))
    bank.update(torch.tensor([3.0]), torch.zeros(1, 4, 2))  # no overwrite unless replace=True (storage.py:62-71)
    lat, msk = bank.get(torch.tensor([2.0, 3.0, 4.0]), "cpu", add_batch_dim=True)
    assert torch.equal(lat, host["bank_get"][0]) and torch.equal(msk, host["bank_get"][1])
    bank.update(torch.tensor([3.0]), torch.zeros(1, 4, 2), replace=True)
    assert float(bank.get(torch.tensor([3.0]), "cpu")[0].abs().sum()) == 0.0
    bank.update(torch.tensor([1.0]), torch.full((1, 4, 2), 2.0))
    lat, ts = bank.get_ordered()
    assert ts.tolist() == [1.0, 3.0] and float(lat[0, 0, 0]) == 2.0


def test_gelu_erfc_form_error_bound():
    """The GEMM epilogue evaluates the reference's exact (erf) GELU as x * Phi(x) with Phi(-|x|) = erfc(|x| / sqrt 2) / 2 through
    Abramowitz-Stegun 7.1.26 (csrc/gemm.cu gelu_erf).  Re-evaluate that form in fp32 with the constants parsed from the source:
    the absolute error against erf-GELU in float64 stays below 1e-6 over |x| <= 12 — the same as the fp32 erf formula."""
    import math
    import re

    import numpy as np

    src = open(os.path.join(ROOT, "actionmesh_b200", "csrc", "gemm.cu")).read()
    body = src[src.index("__device__ __forceinline__ float gelu_erf"):]
    body = body[:body.index("\n}\n")]
    consts = [np.float32(v) for v in re.findall(r"(-?[01]\.\d{9})f", body)]
    assert len(consts) == 5, consts                       # a5 .. a1 of 7.1.26 in Horner order
    assert "0.3275911f" in body
    f = np.float32
    x = np.linspace(-12.0, 12.0, 2_000_001).astype(np.float32)
    ax = np.abs(x)
    t = (f(1.0) / (f(0.3275911 * 0.70710678118654752440) * ax + f(1.0))).astype(np.float32)
    p = (t * consts[0] + consts[1]).astype(np.float32)
    for c in consts[2:]:
        p = (p * t + c).astype(np.float32)
    e = np.exp2((ax * ax * f(-0.5 * 1.4426950408889634)).astype(np.float32)).astype(np.float32)
    q = (f(0.5) * (p * t).astype(np.float32) * e).astype(np.float32)
    g = (x * np.where(x >= 0, f(1.0) - q, q)).astype(np.float32)
    ref = np.array([0.5 * v * (1.0 + math.erf(v / math.sqrt(2.0))) for v in x[::200].astype(np.float64)])
    assert np.abs(g[::200].astype(np.float64) - ref).max() < 1e-6


def test_image_encoder_constructor_contract():
    """B200ImageEncoder keeps the reference's constructor keywords (image_encoder.py:16-36) and refuses what it cannot honour
    at construction time: a hub id / missing directory (no network, no silent default) and an unknown precision."""
    import pytest

    from actionmesh_b200._lib import AmbError
    from actionmesh_b200.image_encoder import B200ImageEncoder

    enc = B200ImageEncoder(pretrained_dino_feature_extractor=None, pretrained_dino_model=None)
    assert enc.precision == "fp32" and enc.image_preprocess_dino is not None
    assert B200ImageEncoder(precision="bf16").precision == "bf16"
    with pytest.raises(AmbError):
        B200ImageEncoder(pretrained_dino_model="facebook/dinov2-large")
    with pytest.raises(AmbError):
        B200ImageEncoder(precision="fp16")
    with pytest.raises(AmbError):
        enc.to("cpu")
