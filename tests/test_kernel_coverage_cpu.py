"""Keeps the GEMM configuration table of tests/kernel_exact.py honest, on the CPU: the denoiser's single-GPU and sharded
launch programs run against a recording fake of ops.gemm / ops.flash_attn, every GEMM call is reduced to its epilogue
signature (output type, bias, activation, scale, residual and whether it aliases the output, out2, row-map shape, norm /
RoPE layout, two A sources, strided output, tile width), and each signature must be one that the exactness tests run.  A
new call site with an untested epilogue fails here."""
import pytest
import torch

import kernel_exact as kx
from actionmesh_b200 import denoiser as dn
from actionmesh_b200 import ops
from oracle import synth


class _Recorder:
    def __init__(self):
        self.signatures = {}

    def gemm(self, a, w, out, *, bias=None, a2=None, residual=None, act=0, col_scale=None, row_map=None, norm=None, out2=None,
             tag="gemm"):
        k = a.shape[1] + (a2.shape[1] if a2 is not None else 0)
        assert a.dtype == w.dtype == torch.bfloat16 and k == w.shape[1] and out.shape[1] == w.shape[0], (a.shape, w.shape, out.shape)
        sig = kx.gemm_signature(a, w, out, bias=bias, a2=a2, residual=residual, act=act, col_scale=col_scale, row_map=row_map,
                                norm=norm, out2=out2)
        self.signatures.setdefault(sig, (tuple(a.shape), tuple(w.shape), tag))
        return out

    def layernorm(self, x, gamma, beta, eps, out=None):
        return out

    def flash_attn(self, q, k, v, o, scale, kv_chunks=1, tag="attn"):
        assert q.shape[-1] in (64, 128) and o.shape == q.shape
        return o

    def timestep_embedding(self, t, channels, out=None, mask=None, rows=None):
        return out

    def add_bias_rows(self, y, bias):
        pass

    def cast_bf16(self, src, out=None):
        return torch.empty(src.shape, dtype=torch.bfloat16) if out is None else out


def _model(monkeypatch, residual_fp32):
    rec = _Recorder()
    for name in ("gemm", "layernorm", "flash_attn", "timestep_embedding", "add_bias_rows", "cast_bf16"):
        monkeypatch.setattr(ops, name, getattr(rec, name))
    d = dict(num_layers=5, num_attention_heads=2, width=256, cross_attention_dim=128, in_channels=64, mlp_ratio=4.0)
    cfg = dn.DenoiserConfig(inflated_layers=(0, 1, 2, 3, 4), **d)
    m = dn.B200Denoiser(cfg, residual_fp32=residual_fp32)
    m._w = m._pack_state_dict(synth.make_state_dict(cfg, 1), torch.device("cpu"))
    m._loaded = True
    return m, rec


def _single_gpu(m):
    B, T, N = 2, 4, 31
    ctx = torch.randn(B, T, 9, 128)
    ctx[0] = 0
    fs = torch.arange(T, dtype=torch.float32)[None].repeat(B, 1)
    st = m.precompute_window(ctx, fs, N)
    m._forward_packed(m._workspace(B, T, N), st, B, T, N, torch.tensor([500.0]), torch.zeros(B * T), n_input_branches=1)


def _sharded(m):
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


@pytest.fixture(scope="module")
def table():
    return kx.table_signatures()


@pytest.mark.parametrize("program", ["single_gpu", "sharded"])
@pytest.mark.parametrize("residual_fp32", [True, False])
def test_denoiser_gemm_epilogues_are_in_the_table(monkeypatch, table, program, residual_fp32):
    m, rec = _model(monkeypatch, residual_fp32)
    (_single_gpu if program == "single_gpu" else _sharded)(m)
    assert rec.signatures
    missing = {sig: where for sig, where in rec.signatures.items() if sig not in table}
    assert not missing, "GEMM epilogues launched without a row in kernel_exact.GEMM_CONFIGS:\n" + "\n".join(
        f"  {where}: {dict(sig)}" for sig, where in missing.items())

