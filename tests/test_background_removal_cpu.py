"""Background removal without a GPU: the fp32 restatement (tests/rmbg_ref.py) against the reference's own BriaRMBG golden,
Otsu against cv2, the component filter on crafted masks, the launch program's GEMM configurations and shapes, BN folding
and the split weight layout, and the argument checks of the new C entry points."""
import ctypes as C

import numpy as np
import pytest
import torch

import kernel_exact as kx
import rmbg_ref
from actionmesh_b200 import background_removal as br
from actionmesh_b200 import ops
from conftest import load_golden
from test_background_removal_gpu import RMBG_GEMM_CONFIGS
from test_kernel_coverage_cpu import _Coverage


def test_restatement_equals_reference_golden():
    g = load_golden("rmbg_tiny.pt")
    image = rmbg_ref.synthetic_frame(*g["frame"], g["frame_seed"])
    out = rmbg_ref.remove_background(rmbg_ref.make_state_dict(g["seed"]), image, g["model_size"], min_size=g["min_size"])
    assert out["soft"].shape == g["soft"].shape
    assert (out["soft"] - g["soft"]).abs().max().item() <= 1e-6
    assert np.array_equal(out["mask"], g["mask"].numpy())
    assert np.array_equal(out["rgba"][..., 3], g["refined"].numpy())
    assert 0.05 < (g["refined"] > 0).float().mean().item() < 0.95, "the golden's refined mask should hold both classes"


def _otsu_cases():
    rng = np.random.default_rng(3)
    cases = {"constant": np.full((17, 23), 91, np.uint8), "zeros": np.zeros((8, 8), np.uint8),
             "two_level": np.where(rng.random((40, 31)) < 0.3, 20, 200).astype(np.uint8),
             "single_pixel_class": np.pad(np.full((1, 1), 255, np.uint8), ((0, 99), (0, 99))),
             "empty_middle": np.concatenate([np.zeros((10, 10), np.uint8), np.full((10, 10), 255, np.uint8)])}
    for i in range(60):
        h, w = rng.integers(1, 90, 2)
        kind = i % 4
        if kind == 0:
            m = rng.integers(0, 256, (h, w))
        elif kind == 1:
            m = np.clip(rng.normal(rng.uniform(40, 200), rng.uniform(2, 60), (h, w)), 0, 255)
        elif kind == 2:
            m = rng.choice(rng.integers(0, 256, rng.integers(2, 5)), (h, w))
        else:
            m = np.where(rng.random((h, w)) < rng.uniform(0.05, 0.95), rng.normal(60, 15, (h, w)), rng.normal(180, 25, (h, w)))
        cases[f"random{i}"] = np.clip(m, 0, 255).astype(np.uint8)
    return cases


@pytest.mark.parametrize("name,mask", list(_otsu_cases().items()))
def test_otsu_restatement_equals_cv2(name, mask):
    t, binary = rmbg_ref.otsu_cv2(mask)
    assert rmbg_ref.otsu_threshold(np.bincount(mask.ravel(), minlength=256)) == t
    assert np.array_equal(binary, np.where(mask > t, 255, 0).astype(np.uint8))


def _blob(n):
    """A 4-connected run of exactly n pixels in a 40-wide strip."""
    m = np.zeros((n // 40 + 1, 40), np.uint8)
    m.ravel()[:n] = 1
    return m


def test_component_filter_crafted():
    m = np.zeros((60, 90), np.uint8)
    for k in range(30):            # a diagonal-only line: one 8-connected component of 30 pixels
        m[k, k + 50] = 1
    m[10:15, 0:40] = _blob(199)[:5, :40]   # exactly 199 pixels: removed
    m[20:26, 0:40] = _blob(200)[:6, :40]   # exactly 200 pixels: kept
    m[55:60, 80:90] = 1                     # a border component of 50 pixels
    out = rmbg_ref.filter_components(m, 30)
    assert out.dtype == np.uint8 and set(np.unique(out)) <= {0, 255}
    assert (out[:30, 50:] > 0).sum() == 30, "diagonal neighbours join one component"
    assert (rmbg_ref.filter_components(m, 31)[:30, 50:] == 0).all()
    out = rmbg_ref.filter_components(m, 200)
    assert (out[10:15] == 0).all() and (out[20:26] > 0).sum() == 200 and (out[55:] == 0).all()
    assert (rmbg_ref.filter_components(m, 50)[55:60, 80:90] == 255).all()


class _RmbgCoverage(_Coverage):
    """The GEMM-recording fake plus shape-checking fakes of the rmbg ops."""

    def __init__(self):
        super().__init__()
        self.shapes = []

    def rmbg_resize_input(self, rgb, out):
        assert rgb.dtype == torch.uint8 and out.dtype == torch.float32 and out.shape[2] == 3
        return out

    def rmbg_im2col_split(self, sources, h, w, out, stride=1, pad=1, dilation=1):
        rows = ops.conv3x3_out(h, stride, pad, dilation) * ops.conv3x3_out(w, stride, pad, dilation)
        for t, c in sources:
            ops._feature_map(t, h, w, c, "source")
        assert out.dtype == torch.bfloat16 and out.shape[0] == rows and out.shape[1] % 192 == 0
        assert 9 * sum(c for _, c in sources) <= out.shape[1] // 3
        return out

    def rmbg_maxpool2(self, src, h, w, c, out):
        ops._feature_map(src, h, w, c, "src")
        ops._feature_map(out, (h + 1) // 2, (w + 1) // 2, c, "out")
        return out

    def rmbg_upsample(self, src, h, w, c, out, oh, ow):
        ops._feature_map(src, h, w, c, "src")
        ops._feature_map(out, oh, ow, c, "out")
        return out

    def rmbg_mask_head(self, feat, h, w, weight, model_size, out_size, work=None):
        ops._feature_map(feat, h, w, 64, "feat")
        assert weight.shape == (577,)
        self.shapes.append(("head", h, w, tuple(model_size), tuple(out_size)))
        work = {} if work is None else work
        work.setdefault("mask", torch.zeros(tuple(out_size), dtype=torch.uint8))
        return work

    def rmbg_refine_rgba(self, rgb, mask, refine=True, min_size=200, out=None, work=None):
        return torch.zeros(*rgb.shape[:2], 4, dtype=torch.uint8)


def _remover_on_cpu(model_size):
    m = br.B200BackgroundRemover(model_input_size=model_size)
    m._w = m._pack_state_dict(rmbg_ref.make_state_dict(0), torch.device("cpu"))
    m._loaded = True
    return m


@pytest.mark.parametrize("model_size,frame", [((1024, 1024), (720, 1280)), ((200, 264), (180, 240))])
def test_launch_program_gemm_configurations_and_shapes(monkeypatch, model_size, frame):
    rec = _RmbgCoverage()
    for name in ("gemm", "rmbg_resize_input", "rmbg_im2col_split", "rmbg_maxpool2", "rmbg_upsample", "rmbg_mask_head",
                 "rmbg_refine_rgba"):
        monkeypatch.setattr(ops, name, getattr(rec, name))
    m = _remover_on_cpu(model_size)
    rgba, _ = m._run(torch.zeros(*frame, 3, dtype=torch.uint8))
    assert rgba.shape == (*frame, 4)
    table = {kx.gemm_signature(c.a, c.w, c.out, **c.kw)
             for c in (kx.build_gemm_case(cfg, 8, "cpu", pad=False) for cfg in RMBG_GEMM_CONFIGS)}
    missing = {sig: sites for sig, sites in rec.signatures.items() if sig not in table}
    assert not missing, f"GEMM configurations without a row in RMBG_GEMM_CONFIGS: {missing}"
    convs = [c for c in rec.calls if c[0] == "gemm"]
    assert len(convs) == len(br.conv_layers())
    hc, wc = (model_size[0] + 1) // 2, (model_size[1] + 1) // 2
    assert rec.shapes == [("head", hc, wc, model_size, frame)]
    # the (N, K) pairs the GPU table runs are exactly the network's
    pairs = {(w[0], w[1]) for _, _, w in convs}
    assert pairs == {(c.n, c.k) for c in RMBG_GEMM_CONFIGS}
    if model_size == (1024, 1024):
        biggest = max(a[0] * a[1] for _, a, _ in convs)
        assert biggest == 512 * 512 * 3 * 1152  # stage1d's rebnconvin: 1.8 GB of bf16


def test_bn_folding_and_split_weight_layout():
    sd = rmbg_ref.make_state_dict(0)
    packed = _remover_on_cpu((64, 64))._w
    for prefix, cin, cout, dil, bn in br.conv_layers()[:: 7] + br.conv_layers()[-1:]:
        key = f"{prefix}.conv_s1" if bn else prefix
        w, b = sd[f"{key}.weight"].double(), sd[f"{key}.bias"].double()
        if bn:
            bp = f"{prefix}.bn_s1"
            s = sd[f"{bp}.weight"].double() / (sd[f"{bp}.running_var"].double() + 1e-5).sqrt()
            w, b = w * s[:, None, None, None], (b - sd[f"{bp}.running_mean"].double()) * s + sd[f"{bp}.bias"].double()
        wp, bp_ = packed[f"{prefix}.w"], packed[f"{prefix}.b"]
        kpad, npad = (9 * cin + 63) // 64 * 64, (cout + 63) // 64 * 64
        assert wp.shape == (npad, 3 * kpad) and wp.dtype == torch.bfloat16 and bp_.shape == (npad,)
        hi, hi2, lo = wp[:, :kpad].float(), wp[:, kpad:2 * kpad].float(), wp[:, 2 * kpad:].float()
        assert torch.equal(hi, hi2)
        rows = w.permute(0, 2, 3, 1).reshape(cout, 9 * cin)          # (O, ky, kx, I) order
        got = hi.double() + lo.double()
        assert (got[:cout, :9 * cin] - rows).abs().max() <= 2.0 ** -16 * rows.abs().max()
        assert (got[cout:] == 0).all() and (got[:, 9 * cin:] == 0).all() and (bp_[cout:] == 0).all()
        assert (bp_[:cout].double() - b).abs().max() <= 1e-6 * b.abs().max()
    s1 = packed["side1"]
    assert torch.equal(s1[:576], sd["side1.weight"][0].permute(1, 2, 0).reshape(-1)) and s1[576] == sd["side1.bias"][0]


def test_pack_refuses_unknown_and_missing_keys():
    sd = dict(rmbg_ref.make_state_dict(0))
    m = br.B200BackgroundRemover(model_input_size=(64, 64))
    with pytest.raises(br.AmbError, match="unexpected"):
        m._pack_state_dict({**sd, "outconv.weight": torch.zeros(1)}, torch.device("cpu"))
    del sd["stage3.rebnconv2.bn_s1.running_var"]
    with pytest.raises(br.AmbError, match="missing"):
        m._pack_state_dict(sd, torch.device("cpu"))
    sd = {k: v for k, v in rmbg_ref.make_state_dict(0).items() if not k.startswith(("side2", "side5")) and "num_batches" not in k}
    m._pack_state_dict(sd, torch.device("cpu"))  # the unused heads and counters may be absent


def test_rmbg_entry_points_validate_arguments(amb_lib):
    fake, odd = 1 << 20, (1 << 20) + 1
    calls = [
        (amb_lib.amb_rmbg_resize_input, (None, 4, 4, fake, 8, 8, None), b"null pointer"),
        (amb_lib.amb_rmbg_resize_input, (fake, 0, 4, fake, 8, 8, None), b"bad sizes"),
        (amb_lib.amb_rmbg_resize_input, (fake, 4, 4, odd, 8, 8, None), b"aligned"),
        (amb_lib.amb_rmbg_im2col_split, (fake, 3, 2, None, 0, 0, 8, 8, 1, 1, 1, 64, fake, 192, None), b"bad channels"),
        (amb_lib.amb_rmbg_im2col_split, (fake, 8, 8, None, 0, 0, 8, 8, 1, 1, 1, 64, fake, 192, None), b"bad k_pad"),
        (amb_lib.amb_rmbg_im2col_split, (fake, 3, 3, None, 0, 0, 8, 8, 1, 1, 1, 48, fake, 192, None), b"bad k_pad"),
        (amb_lib.amb_rmbg_im2col_split, (fake, 3, 3, None, 0, 0, 8, 8, 1, 1, 1, 64, fake, 100, None), b"bad k_pad"),
        (amb_lib.amb_rmbg_im2col_split, (fake, 3, 3, None, 0, 0, 8, 8, 3, 1, 1, 64, fake, 192, None), b"bad stride"),
        (amb_lib.amb_rmbg_im2col_split, (fake, 3, 3, None, 0, 0, 4, 4, 1, 0, 8, 64, fake, 192, None), b"too small"),
        (amb_lib.amb_rmbg_im2col_split, (fake, 3, 3, None, 5, 5, 8, 8, 1, 1, 1, 64, fake, 192, None), b"null pointer"),
        (amb_lib.amb_rmbg_im2col_split, (odd, 3, 3, None, 0, 0, 8, 8, 1, 1, 1, 64, fake, 192, None), b"misaligned"),
        (amb_lib.amb_rmbg_maxpool2, (fake, 3, 8, 8, 4, fake, 4, None), b"bad geometry"),
        (amb_lib.amb_rmbg_maxpool2, (fake, 4, 8, 8, 4, None, 4, None), b"null pointer"),
        (amb_lib.amb_rmbg_upsample, (fake, 4, 8, 8, 4, fake, 4, 0, 5, None), b"bad geometry"),
        (amb_lib.amb_rmbg_upsample, (fake, 4, 8, 8, 4, odd, 4, 5, 5, None), b"misaligned"),
        (amb_lib.amb_rmbg_mask_head, (fake, 32, 8, 8, fake, fake, 16, 16, fake, 20, 20, fake, fake, fake, None), b"pixel stride"),
        (amb_lib.amb_rmbg_mask_head, (fake + 4, 64, 8, 8, fake, fake, 16, 16, fake, 20, 20, fake, fake, fake, None), b"misaligned"),
        (amb_lib.amb_rmbg_mask_head, (fake, 64, 8, 8, fake, fake, 16, 0, fake, 20, 20, fake, fake, fake, None), b"bad sizes"),
        (amb_lib.amb_rmbg_mask_head, (fake, 64, 8, 8, None, fake, 16, 16, fake, 20, 20, fake, fake, fake, None), b"null pointer"),
        (amb_lib.amb_rmbg_refine_rgba, (fake, fake, 8, 8, 1, 200, None, fake, fake, fake, None), b"null pointer"),
        (amb_lib.amb_rmbg_refine_rgba, (fake, fake, 8, 8, 1, 200, fake, fake, fake, odd, None), b"misaligned"),
        (amb_lib.amb_rmbg_refine_rgba, (fake, fake, -1, 8, 0, 200, None, None, None, fake, None), b"bad size"),
        (amb_lib.amb_rmbg_refine_rgba, (fake, fake, 8, 8, 2, 200, fake, fake, fake, fake, None), b"refine must be"),
        (amb_lib.amb_rmbg_refine_rgba, (fake, fake, 1 << 16, 1 << 15, 0, 200, None, None, None, fake, None), b"bad size"),
    ]
    for fn, args, msg in calls:
        rc = fn(*args)
        assert rc < 0, (fn.__name__, args)
        assert msg in amb_lib.amb_last_error(), (fn.__name__, args, amb_lib.amb_last_error())


def test_gemm_refuses_unknown_activation(amb_lib):
    from actionmesh_b200 import _lib

    g = _lib.GemmArgs()
    g.a, g.w, g.c = 16, 16, 16
    g.m, g.n, g.k = 128, 64, 64
    g.lda = g.ldw = g.ldc = 64
    g.act = 3
    assert amb_lib.amb_gemm_bf16(C.byref(g), None) < 0 and b"unknown activation 3" in amb_lib.amb_last_error()


def test_remover_refuses_cpu_and_bad_images():
    m = br.B200BackgroundRemover(model_input_size=(64, 64))
    with pytest.raises(br.AmbError, match="no CPU fallback"):
        m.to("cpu")
    with pytest.raises(br.AmbError, match="model_input_size"):
        br.B200BackgroundRemover(model_input_size=(0, 64))
    with pytest.raises(br.AmbError):
        m._run(torch.zeros(8, 8, 3, dtype=torch.uint8))  # weights not loaded
