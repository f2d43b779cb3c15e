"""Structural CPU test of the host launch programs (no GPU, no arithmetic): `B200Denoiser._forward_packed` (single GPU) and
the staggered per-branch programs of the frame-sharded window, `B200Autoencoder.forward`, `B200TripoSGVAE.prepare` / `query`
/ `encode_points` and `B200ImageEncoder.encode_pixel_values` are executed against shape/dtype-checking fakes of the C-ABI
wrappers in actionmesh_b200.ops, with weights packed on the CPU.  Catches slicing / buffer-plumbing / generator-flow mistakes in the host code
that would otherwise only show on a GPU box; the numerics are covered by the -m gpu parity tests."""
import pytest
import torch

from actionmesh_b200 import denoiser as dn
from actionmesh_b200 import ops
from actionmesh_b200.autoencoder import AutoencoderConfig, B200Autoencoder
from actionmesh_b200.image_encoder import B200ImageEncoder
from actionmesh_b200.triposg_vae import B200TripoSGVAE
from oracle import synth


class _Recorder:
    def __init__(self):
        self.calls = []

    def gemm(self, a, w, out, *, bias=None, a2=None, residual=None, act=0, col_scale=None, row_map=None, norm=None, out2=None, tag="gemm"):
        k = a.shape[1] + (a2.shape[1] if a2 is not None else 0)
        assert a.dtype == w.dtype == torch.bfloat16 and k == w.shape[1] and out.shape[1] == w.shape[0], (a.shape, w.shape, out.shape)
        assert a.stride(1) == 1 and w.stride(1) == 1 and out.stride(1) == 1
        if a2 is not None:
            assert a2.shape[0] == a.shape[0]
        if row_map is None:
            assert out.shape[0] >= a.shape[0]
        else:
            grp, stride, off = row_map
            last = (a.shape[0] - 1) // grp * stride + (a.shape[0] - 1) % grp + off
            assert last < out.shape[0], (row_map, a.shape, out.shape)
        if residual is not None:
            assert residual.shape[1] == out.shape[1] and residual.shape[0] >= a.shape[0]
        if bias is not None:
            assert bias.dtype == torch.float32 and bias.numel() == w.shape[0]
        if norm is not None and norm.get("rope_cols", 0):
            n_pos = (a.shape[0] + norm["rows_per_pos"] - 1) // norm["rows_per_pos"]
            assert norm["cos"].shape[0] >= n_pos and norm["cos"].shape == norm["sin"].shape, (norm["cos"].shape, n_pos)
        if out2 is not None:
            assert out2.dtype == torch.bfloat16 and out2.shape == out.shape and out.dtype == torch.float32
            self.calls.append(("gemm_out2", tuple(out2.shape)))
        self.calls.append(("gemm", tuple(a.shape), tuple(w.shape)))
        return out

    def layernorm(self, x, gamma, beta, eps, out=None):
        assert out is not None and out.shape == x.shape and gamma.numel() == x.shape[1]
        self.calls.append(("ln", tuple(x.shape)))
        return out

    def flash_attn(self, q, k, v, o, scale, kv_chunks=1, tag="attn"):
        if kv_chunks == 1:
            assert q.dim() == k.dim() == 4 and k.shape == v.shape and q.shape[0] == k.shape[0] and q.shape[2:] == k.shape[2:]
        else:
            assert k.dim() == 5 and k.shape[1] == kv_chunks and k.shape == v.shape and q.shape[2:] == k.shape[3:]
        assert o.shape == q.shape
        self.calls.append((tag, tuple(q.shape), tuple(k.shape)))
        return o

    def timestep_embedding(self, t, channels, out=None, mask=None, rows=None):
        assert out.shape == (rows, channels)
        return out

    def add_bias_rows(self, y, bias):
        assert bias.numel() == y.shape[1]
        self.calls.append(("bias_rows", tuple(y.shape)))

    def cast_bf16(self, src, out=None):
        if out is None:
            out = torch.empty(src.shape, dtype=torch.bfloat16)
        assert out.numel() == src.numel() and src.dtype == torch.float32 and out.dtype == torch.bfloat16
        self.calls.append(("cast", tuple(src.shape)))
        return out

    def split3(self, src, out, seg=None, weight=False):
        rows, cols = src.shape
        assert src.dtype == torch.float32 and out.dtype == torch.bfloat16 and out.shape[0] >= rows and out.shape[1] == 3 * cols
        assert cols % (seg or cols) == 0
        self.calls.append(("split3", tuple(src.shape)))
        return out

    def point_embedding(self, points, num_freqs, include_pi, kpad):
        assert points.dtype == torch.float32 and points.dim() == 2
        assert kpad % 64 == 0 and kpad >= 3 * (2 * num_freqs + 1) + points.shape[1] - 3
        return torch.empty(points.shape[0], kpad, dtype=torch.float32)

    def alpha_rows(self, source_alpha, target_alpha, size, out_rows):
        assert out_rows.dtype == torch.float32 and out_rows.dim() == 2 and out_rows.shape[1] == 2 * size
        self.calls.append(("alpha_rows", tuple(out_rows.shape)))

    def softmax_split3(self, scores, n, scale, out):
        rows, n_pad = scores.shape
        assert scores.dtype == torch.float32 and n <= n_pad and out.shape == (rows, 3 * n_pad)
        self.calls.append(("softmax_split3", tuple(scores.shape)))
        return out

    def displacement_out(self, logits, out_dim, out):
        assert logits.dtype == out.dtype == torch.float32 and out.numel() == logits.shape[0] * out_dim
        self.calls.append(("displacement_out", tuple(out.shape)))
        return out

    def attn_small_f32(self, qkv, frames, seq, heads, scale, out, tag="attn_small"):
        assert qkv.dtype == out.dtype == torch.float32
        assert qkv.shape == (frames * seq, 3 * heads * 64) and out.shape == (frames * seq, heads * 64)
        self.calls.append((tag, (frames, seq, heads, 64), (frames, seq, heads, 64)))
        return out

    def patchify(self, pixels, patch, kpad, out=None):
        T, C, H, W = pixels.shape
        assert C == 3 and pixels.dtype == torch.float32 and kpad >= 3 * patch * patch
        return torch.empty(T * (H // patch) * (W // patch), kpad, dtype=torch.bfloat16)


def _recorder(monkeypatch):
    rec = _Recorder()
    for name in ("gemm", "layernorm", "flash_attn", "timestep_embedding", "add_bias_rows", "cast_bf16", "split3",
                 "point_embedding", "alpha_rows", "softmax_split3", "displacement_out", "attn_small_f32", "patchify"):
        monkeypatch.setattr(ops, name, getattr(rec, name))
    return rec


def _load_on_cpu(m):
    """init_random_'s weights, packed on the CPU (load_state_dict needs a CUDA device)."""
    m.load_state_dict = lambda sd: setattr(m, "_w", m._pack_state_dict(sd, torch.device("cpu")))
    m.init_random_()
    m._loaded = True
    return m


def _model(monkeypatch, residual_fp32=True):
    rec = _recorder(monkeypatch)
    d = dict(num_layers=5, num_attention_heads=2, width=256, cross_attention_dim=128, in_channels=64, mlp_ratio=4.0)
    cfg = dn.DenoiserConfig(inflated_layers=(0, 1, 2, 3, 4), **d)
    m = dn.B200Denoiser(cfg, residual_fp32=residual_fp32)
    m._w = m._pack_state_dict(synth.make_state_dict(cfg, 1), torch.device("cpu"))
    m._loaded = True
    return m, rec, cfg


@pytest.mark.parametrize("residual_fp32", [True, False])
def test_single_gpu_program(monkeypatch, residual_fp32):
    m, rec, cfg = _model(monkeypatch, residual_fp32)
    B, T, N = 2, 4, 31
    ctx = torch.randn(B, T, 9, 128)
    ctx[0] = 0
    fs = torch.arange(T, dtype=torch.float32)[None].repeat(B, 1)
    st = m.precompute_window(ctx, fs, N)
    assert st.ctx_zero == [True, False]
    ws = m._workspace(B, T, N)
    pred = m._forward_packed(ws, st, B, T, N, torch.tensor([500.0]), torch.zeros(B * T), n_input_branches=1)
    assert pred.shape == (B * T * (N + 1), 64)
    attn = [c for c in rec.calls if c[0] == "attn_self"]
    assert len(attn) == cfg.num_layers and all(c[1] == (B, T * (N + 1), 2, 128) for c in attn)
    assert sum(1 for c in rec.calls if c[0] == "attn_cross") == cfg.num_layers      # only the non-zero-context branch
    assert sum(1 for c in rec.calls if c[0] == "bias_rows") == cfg.num_layers
    # fp32 residual stream: one bf16 operand copy per skip push and per skip pop, written as the second output of the
    # producing GEMM (no separate cast pass); none with the bf16 stream
    assert not [c for c in rec.calls if c[0] == "cast" and c[1] == (B * T * (N + 1), cfg.width)]
    assert len([c for c in rec.calls if c[0] == "gemm_out2"]) == (2 * (cfg.num_layers // 2) if residual_fp32 else 0)
    assert ws["h"].dtype == (torch.float32 if residual_fp32 else torch.bfloat16)


def test_sharded_branch_programs_interleave(monkeypatch):
    m, rec, cfg = _model(monkeypatch)
    order = []

    class _Work:
        def __init__(self, tag):
            self.tag = tag

        def wait(self):
            order.append(("wait", self.tag))

    world, B, T_all, N = 2, 2, 4, 31
    T = T_all // world

    class Shard:
        group = None

        @staticmethod
        def all_gather_kv(out, inp, channel=0):
            assert out.shape[0] == world * inp.shape[0] and out.shape[1] == inp.shape[1]
            order.append(("gather", out.data_ptr()))
            return _Work(out.data_ptr())

    Shard.world, Shard.rank = world, 0
    ctx = torch.randn(B, T_all, 9, 128)
    ctx[0] = 0
    fs = torch.arange(T_all, dtype=torch.float32)[None].repeat(B, 1)
    st = m.precompute_window(ctx, fs, N, frame_slice=slice(0, T))
    ws = m._workspace(B, T, N, world=world)
    pred = m._forward_packed(ws, st, B, T, N, torch.tensor([500.0]), torch.zeros(B * T), n_input_branches=1, shard=Shard)
    assert pred.shape == (B * T * (N + 1), 64)
    gathers = [o for o in order if o[0] == "gather"]
    assert len(gathers) == B * cfg.num_layers
    # staggering: between a branch's gather and its wait, the OTHER branch's gather/wait is issued (except at the very start)
    tags = [o for o in order]
    for i in range(len(tags) - 1):
        if tags[i][0] == "gather" and i > 0:
            assert not (tags[i + 1][0] == "wait" and tags[i + 1][1] == tags[i][1]), "a gather was waited on immediately"
    attn = [c for c in rec.calls if c[0] == "attn_self"]
    assert len(attn) == B * cfg.num_layers and all(c[1] == (1, T * (N + 1), 2, 128) and c[2][:3] == (1, world, T * (N + 1)) for c in attn)


def test_autoencoder_program(monkeypatch):
    rec = _recorder(monkeypatch)
    cfg = AutoencoderConfig(width=256, num_layers=2, num_attention_heads=2, temporal_context_size=4)
    m = _load_on_cpu(B200Autoencoder(cfg))
    B, T, N, V, T_out = 2, 4, 15, 20, 3
    out = m.forward(torch.randn(B, T, N, 64), torch.arange(T, dtype=torch.float32)[None].repeat(B, 1) + 3,
                    torch.full((B,), 0.25), torch.rand(B, T_out), torch.randn(B, V, 6))
    assert out.shape == (B, T_out, V, 3) and out.dtype == torch.float32
    trunk = [c for c in rec.calls if c[0] == "s2_attn"]
    assert len(trunk) == B * T_out * cfg.num_layers and all(c[1] == (1, T * (N + 1), 2, 128) for c in trunk)
    assert sum(1 for c in rec.calls if c[0] == "softmax_split3") == B * T_out * cfg.num_attention_heads
    assert sum(1 for c in rec.calls if c[0] == "alpha_rows") == B * T_out
    assert sum(1 for c in rec.calls if c[0] == "displacement_out") == B * T_out


def test_triposg_vae_programs(monkeypatch):
    rec = _recorder(monkeypatch)
    m = _load_on_cpu(B200TripoSGVAE(width_decoder=256, num_attention_heads=2, num_layers_decoder=2, width_encoder=256,
                                    num_layers_encoder=2))
    assert m._has_encoder
    N, P, chunk = 33, 50, 20
    ctx = m.prepare(torch.randn(N, 64))
    assert ctx.kv.shape == (N, 2 * 256) and ctx.k.shape == ctx.v.shape == (1, N, 2, 128)
    assert [c[1] for c in rec.calls if c[0] == "vae_trunk_attn"] == [(1, N, 2, 128)] * 2
    assert m.query(ctx, torch.randn(P, 3), chunk=chunk).shape == (P, 64)
    assert [c[1:] for c in rec.calls if c[0] == "vae_query_attn"] == [((1, m_, 2, 128), (1, N, 2, 128)) for m_ in (20, 20, 10)]
    n_kv, n_q = 40, 16
    assert m.encode_points(torch.randn(n_kv, 6), torch.randn(n_q, 6)).shape == (n_q, 2 * 64)
    enc = [c[1:] for c in rec.calls if c[0] == "vae_encoder_attn"]
    assert enc == [((1, n_q, 2, 128), (1, n_kv, 2, 128))] + [((1, n_q, 2, 128), (1, n_q, 2, 128))] * 2


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_image_encoder_program(monkeypatch, precision):
    rec = _recorder(monkeypatch)
    m = _load_on_cpu(B200ImageEncoder(hidden_size=256, num_layers=2, num_heads=4, image_size=28, precision=precision))
    T, L = 3, 1 + 2 * 2
    out = m.encode_pixel_values(torch.randn(T, 3, 28, 28))
    assert out.shape == (T, L, 256) and out.dtype == torch.float32
    attn = [c[1] for c in rec.calls if c[0] == "attn_dino"]
    assert attn == [(T, L, 4, 64)] * 2
