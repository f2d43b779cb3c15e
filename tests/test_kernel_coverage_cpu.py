"""Keeps the kernel-level test tables honest, on the CPU: every model's launch programs (the denoiser single-GPU and
sharded, Stage II's autoencoder, the TripoSG VAE's prepare / query / encode_points, DinoV2 at fp32 and bf16, TripoSG's DiT)
run against a recording fake of the C-ABI wrappers, and every call is reduced to the configuration a kernel-level test has
to have exercised:
  * ops.gemm -> its epilogue signature (output type, bias, activation, scale, residual and whether it aliases the output,
    out2, row-map shape, norm / RoPE layout, two A sources, strided output, tile width), which must be a row of
    kernel_exact.GEMM_CONFIGS (run by test_kernel_exactness_gpu and test_gemm_paths_gpu);
  * ops.split3 / ops.softmax_split3 / ops.attn_small_f32 -> a case of split_exact (run by test_fp32_grade_gpu).
A new call site with an untested configuration fails here."""
import pytest
import torch

import kernel_exact as kx
import split_exact as sx
from actionmesh_b200 import denoiser as dn
from actionmesh_b200 import ops
from actionmesh_b200.autoencoder import AutoencoderConfig, B200Autoencoder
from actionmesh_b200.image_encoder import B200ImageEncoder
from actionmesh_b200.stage0 import B200TripoSGDiT
from actionmesh_b200.triposg_vae import B200TripoSGVAE
from oracle import synth
from test_launch_program_cpu import _load_on_cpu, _Recorder


class _Coverage(_Recorder):
    """The shape-checking fake of test_launch_program_cpu, recording the configuration of every call: signature ->
    the distinct (operand shapes, tag) that launched it."""

    def __init__(self):
        super().__init__()
        self.signatures = {}
        self.kernels = {}

    def _note(self, table, sig, where):
        sites = table.setdefault(sig, [])
        if where not in sites:
            sites.append(where)

    def gemm(self, a, w, out, *, tag="gemm", **kw):
        super().gemm(a, w, out, tag=tag, **kw)
        self._note(self.signatures, kx.gemm_signature(a, w, out, **kw), (tag, tuple(a.shape), tuple(w.shape), tuple(out.shape)))
        return out

    def split3(self, src, out, seg=None, weight=False):
        super().split3(src, out, seg, weight)
        self._note(self.kernels, sx.split3_signature(src, out, seg, weight), (tuple(src.shape), seg))
        return out

    def softmax_split3(self, scores, n, scale, out):
        super().softmax_split3(scores, n, scale, out)
        self._note(self.kernels, sx.softmax_signature(scores, n), (tuple(scores.shape), n))
        return out

    def attn_small_f32(self, qkv, frames, seq, heads, scale, out, tag="attn_small"):
        super().attn_small_f32(qkv, frames, seq, heads, scale, out, tag=tag)
        self._note(self.kernels, sx.attn_small_signature(qkv, out, heads), (tag, frames, seq, heads))
        return out


def _recorder(monkeypatch) -> _Coverage:
    rec = _Coverage()
    for name in ("gemm", "layernorm", "flash_attn", "timestep_embedding", "add_bias_rows", "cast_bf16", "split3",
                 "point_embedding", "alpha_rows", "softmax_split3", "displacement_out", "attn_small_f32", "patchify"):
        monkeypatch.setattr(ops, name, getattr(rec, name))
    return rec


_DENOISER = dict(num_layers=5, num_attention_heads=2, width=256, cross_attention_dim=128, in_channels=64, mlp_ratio=4.0)


def _denoiser(residual_fp32):
    cfg = dn.DenoiserConfig(inflated_layers=(0, 1, 2, 3, 4), **_DENOISER)
    m = dn.B200Denoiser(cfg, residual_fp32=residual_fp32)
    m._w = m._pack_state_dict(synth.make_state_dict(cfg, 1), torch.device("cpu"))
    m._loaded = True
    return m


def _denoiser_single_gpu(residual_fp32):
    m = _denoiser(residual_fp32)
    B, T, N = 2, 4, 31
    ctx = torch.randn(B, T, 9, 128)
    ctx[0] = 0
    fs = torch.arange(T, dtype=torch.float32)[None].repeat(B, 1)
    st = m.precompute_window(ctx, fs, N)
    m._forward_packed(m._workspace(B, T, N), st, B, T, N, torch.tensor([500.0]), torch.zeros(B * T), n_input_branches=1)


def _denoiser_sharded(residual_fp32):
    m = _denoiser(residual_fp32)
    world, B, T_all, N = 2, 2, 4, 31
    T = T_all // world

    class _Work:
        def wait(self):
            pass

    class Shard:
        group = None

        @staticmethod
        def all_gather_kv(out, inp, channel=0):
            return _Work()

    Shard.world, Shard.rank = world, 0
    ctx = torch.randn(B, T_all, 9, 128)
    ctx[0] = 0
    fs = torch.arange(T_all, dtype=torch.float32)[None].repeat(B, 1)
    st = m.precompute_window(ctx, fs, N, frame_slice=slice(0, T))
    m._forward_packed(m._workspace(B, T, N, world=world), st, B, T, N, torch.tensor([500.0]), torch.zeros(B * T),
                      n_input_branches=1, shard=Shard)


def _autoencoder():
    """Width 1024 (the default): the query path's split GEMMs have K = 3072 or 12 288 and N a multiple of 256, so they
    run on the cooperative tiles; R = 4 x 11 = 44 keys pad to Rp = 64, so the softmax has padding columns and the score
    and V-transpose GEMMs have N = Rp = 64 mod 128 and run on BN = 64 tiles, as at the default window (R = 32 784,
    Rp = 32 832)."""
    cfg = AutoencoderConfig(width=1024, num_layers=1, num_attention_heads=8, temporal_context_size=4)
    m = _load_on_cpu(B200Autoencoder(cfg))
    B, T, N, V, T_out = 1, 4, 10, 20, 2
    m.forward(torch.randn(B, T, N, 64), torch.arange(T, dtype=torch.float32)[None].repeat(B, 1),
              torch.full((B,), 0.25), torch.rand(B, T_out), torch.randn(B, V, 6))


def _triposg_vae():
    m = _load_on_cpu(B200TripoSGVAE(width_decoder=256, num_attention_heads=2, num_layers_decoder=2, width_encoder=256,
                                    num_layers_encoder=2))
    ctx = m.prepare(torch.randn(33, 64))
    m.query(ctx, torch.randn(50, 3), chunk=20)
    m.encode_points(torch.randn(40, 6), torch.randn(16, 6))


def _image_encoder(precision):
    """DinoV2-L's width: the fp32 path's split GEMMs (K = 3072 / 12 288) run cooperative."""
    m = _load_on_cpu(B200ImageEncoder(hidden_size=1024, num_layers=1, num_heads=16, image_size=28, precision=precision))
    m.encode_pixel_values(torch.randn(3, 3, 28, 28))


def _triposg_dit():
    cfg = dn.DenoiserConfig(num_tokens_nominal=2048, temporal_context_size=1, inflated_layers=(), **_DENOISER)
    m = B200TripoSGDiT(num_attention_heads=2, width=256, in_channels=64, num_layers=5, cross_attention_dim=128)
    m._w = dn.B200Denoiser._pack_state_dict(m, synth.make_state_dict(cfg, 1), torch.device("cpu"))
    m._loaded = True
    B, N = 2, 31
    m.forward(torch.randn(B, N, 64), torch.tensor([500.0, 500.0]), torch.randn(B, 9, 128))


PROGRAMS = {
    "denoiser_single_gpu_f32res": lambda: _denoiser_single_gpu(True),
    "denoiser_single_gpu_bf16res": lambda: _denoiser_single_gpu(False),
    "denoiser_sharded_f32res": lambda: _denoiser_sharded(True),
    "denoiser_sharded_bf16res": lambda: _denoiser_sharded(False),
    "autoencoder": _autoencoder,
    "triposg_vae": _triposg_vae,
    "image_encoder_fp32": lambda: _image_encoder("fp32"),
    "image_encoder_bf16": lambda: _image_encoder("bf16"),
    "triposg_dit": _triposg_dit,
}


@pytest.fixture(scope="module")
def table():
    return kx.table_signatures()


@pytest.mark.parametrize("program", list(PROGRAMS))
def test_gemm_epilogues_are_in_the_table(monkeypatch, table, program):
    rec = _recorder(monkeypatch)
    PROGRAMS[program]()
    assert rec.signatures
    missing = {sig: where for sig, where in rec.signatures.items() if sig not in table}
    assert not missing, "GEMM epilogues launched without a row in kernel_exact.GEMM_CONFIGS:\n" + "\n".join(
        f"  {dict(sig)}\n    launched by (tag, a, w, out): {where}" for sig, where in missing.items())


@pytest.mark.parametrize("program", list(PROGRAMS))
def test_fp32_grade_calls_are_in_the_table(monkeypatch, program):
    rec = _recorder(monkeypatch)
    PROGRAMS[program]()
    missing = {sig: where for sig, where in rec.kernels.items() if sig not in sx.RUN_SIGNATURES}
    assert not missing, "split3 / softmax_split3 / attn_small_f32 calls without a case in split_exact:\n" + "\n".join(
        f"  {sig}: {where}" for sig, where in missing.items())


def test_programs_reach_the_production_paths(monkeypatch):
    """The recorded programs launch what the tables have to cover: Stage II's score and V-transpose GEMMs on BN = 64
    tiles, split GEMMs on the cooperative tiles (N a multiple of 256, K > 2048), every kind of fp32-grade call."""
    rec = _recorder(monkeypatch)
    _autoencoder()
    _image_encoder("fp32")
    sites = [w for ws in rec.signatures.values() for w in ws]
    assert any(t == "s2_q" and w[0] % 128 == 64 and w[1] == 384 for t, a, w, o in sites), "no BN = 64 score GEMM"
    assert any(t == "s2_q" and w[0] % 128 == 64 and a[0] == 1024 for t, a, w, o in sites), "no BN = 64 V-transpose GEMM"
    assert any(w[0] % 256 == 0 and w[1] == 3 * 4096 for t, a, w, o in sites), "no cooperative split ff2 GEMM"
    want = {("split3", p, s) for p in ("activation", "weight") for s in ("seg == cols", "seg < cols")}
    want |= {("softmax_split3", "n < n_pad"), ("attn_small_f32", "dense strides")}
    assert want <= set(rec.kernels), sorted(rec.kernels)
