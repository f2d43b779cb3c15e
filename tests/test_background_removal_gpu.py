"""Background removal on the GPU: the rmbg kernels bit for bit against restatements, the ReLU GEMM rows on exact operands,
the network against the fp32 oracle (and 10x closer than the oracle with cuDNN TF32), the end-to-end RGBA against the CPU
refinement, the valid-alpha pass-through and the pipeline seam."""
from __future__ import annotations

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import kernel_exact as kx
from actionmesh_b200.background_removal import conv_layers

_pad64 = lambda n: (n + 63) // 64 * 64


def _network_gemm_configs() -> list:
    """One exact-grid GEMM configuration per (N, K, epilogue) the network launches: conv_in (bias), REBNCONV (bias + ReLU)
    and each RSU's rebnconv1d (bias + ReLU + the fp32 hxin residual); fp32 output, K = 3 K_pad (the split operand)."""
    seen, out = set(), []
    for prefix, cin, cout, _, bn in conv_layers():
        n, k = _pad64(cout), 3 * _pad64(9 * cin)
        act, res = (2, "other" if prefix.endswith("rebnconv1d") else None) if bn else (0, None)
        if (n, k, act, res) in seen:
            continue
        seen.add((n, k, act, res))
        name = f"rmbg_n{n}_k{k}_" + ("bias" if not act else "bias_relu_res" if res else "bias_relu")
        out.append(kx.GemmConfig(name, n, k, out="f32", bias=True, act=act, residual=res, res="f32"))
    return out


RMBG_GEMM_CONFIGS = _network_gemm_configs()
gpu = pytest.mark.gpu


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda")


# ---- the ReLU GEMM rows -----------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("cfg", RMBG_GEMM_CONFIGS, ids=lambda c: c.name)
@pytest.mark.parametrize("pad", [False, True])
def test_relu_gemm_rows_exact(cfg, pad):
    from actionmesh_b200 import ops

    dev = _cuda()
    m = 1000
    case = kx.build_gemm_case(cfg, m, dev, seed=cfg.n + cfg.k, pad=pad)
    case.call(ops.gemm)
    torch.cuda.synchronize()
    acc = case.a.double() @ case.w.double().t() + case.kw["bias"].double()
    if cfg.act == 2:
        acc = acc.clamp_min(0.0)          # kernel_exact's reference treats any act as GELU: ReLU is applied here
    if case.res_values is not None:
        acc = acc + case.res_values.double()
    kx.compare(case.out_buf[:m, :cfg.n], acc, None, cfg.name)
    kx.int_view(case.out_buf)[:m, :cfg.n] = kx.NAN_F32
    assert kx.is_untouched(case.out_buf), f"{cfg.name}: wrote outside its rows / columns"


# ---- kernels bit for bit ----------------------------------------------------------------------------------------------------
def _feature(h, w, c, ps, dev, gen, scale=1.0):
    """(h * w, ps) fp32 feature map whose padding columns hold NaN (a read past c would show)."""
    t = torch.full((h * w, ps), float("nan"), device=dev)
    t[:, :c] = torch.randn(h * w, c, generator=gen, device=dev) * scale
    return t


def _im2col_fp32(srcs, h, w, stride, pad, dil, kpad):
    x = torch.cat([t[:, :c].reshape(1, h, w, c).permute(0, 3, 1, 2) for t, c in srcs], 1)
    cols = F.unfold(x, 3, dilation=dil, padding=pad, stride=stride)          # (1, C * 9, L), (c, ky, kx)
    ct = x.shape[1]
    cols = cols[0].reshape(ct, 9, -1).permute(2, 1, 0).reshape(-1, 9 * ct)   # rows, (ky, kx, c)
    out = torch.zeros(cols.shape[0], kpad, device=x.device)
    out[:, :9 * ct] = cols
    return out


@gpu
@pytest.mark.parametrize("stride,dil,two,ps,c0,c1,hw", [
    (2, 1, False, 3, 3, 0, (37, 52)),      # conv_in: stride 2, padding 1, K = 27 -> 64
    (1, 1, False, 64, 32, 0, (33, 20)),    # a padded GEMM output read in place
    (1, 2, True, 64, 16, 16, (21, 30)),    # two sources, K = 288 -> 320
    (1, 4, False, 128, 128, 0, (19, 17)),
    (1, 8, True, 512, 256, 256, (18, 18)),
    (1, 1, True, 64, 64, 64, (9, 7)),
])
def test_im2col_split_equals_split3_of_im2col(stride, dil, two, ps, c0, c1, hw):
    from actionmesh_b200 import ops

    dev = _cuda()
    gen = torch.Generator(device=dev).manual_seed(stride * 100 + dil + c0)
    h, w = hw
    srcs = [(_feature(h, w, c0, ps, dev, gen), c0)] + ([(_feature(h, w, c1, ps + 64, dev, gen), c1)] if two else [])
    pad = dil
    kpad = _pad64(9 * (c0 + c1))
    rows = ops.conv3x3_out(h, stride, pad, dil) * ops.conv3x3_out(w, stride, pad, dil)
    buf = torch.full((rows, 3 * kpad + 64), -7.0, dtype=torch.bfloat16, device=dev)
    got = ops.rmbg_im2col_split(srcs, h, w, buf[:, :3 * kpad], stride=stride, pad=pad, dilation=dil)
    want = ops.split3(_im2col_fp32(srcs, h, w, stride, pad, dil, kpad), torch.empty(rows, 3 * kpad, dtype=torch.bfloat16,
                                                                                      device=dev), seg=kpad)
    torch.cuda.synchronize()
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))
    assert (buf[:, 3 * kpad:] == -7.0).all()


@gpu
@pytest.mark.parametrize("h,w,c,ps", [(8, 8, 64, 64), (13, 7, 32, 64), (25, 33, 16, 64), (1, 5, 3, 3), (100, 132, 512, 512)])
def test_maxpool_equals_torch_ceil_mode(h, w, c, ps):
    from actionmesh_b200 import ops

    dev = _cuda()
    x = _feature(h, w, c, ps, dev, torch.Generator(device=dev).manual_seed(h * w))
    oh, ow = (h + 1) // 2, (w + 1) // 2
    got = ops.rmbg_maxpool2(x, h, w, c, torch.empty(oh * ow, c, device=dev))
    want = F.max_pool2d(x[:, :c].reshape(1, h, w, c).permute(0, 3, 1, 2), 2, 2, ceil_mode=True)
    assert torch.equal(got.view(oh, ow, c), want[0].permute(1, 2, 0))


@gpu
@pytest.mark.parametrize("h,w,oh,ow", [(4, 5, 7, 9), (7, 9, 13, 17), (13, 17, 25, 33), (256, 256, 512, 512), (512, 512, 1024, 1024),
                                       (1024, 1024, 300, 457), (100, 132, 200, 264), (1, 1, 3, 2)])
def test_bilinear_equals_restatement_and_torch(h, w, oh, ow):
    import rmbg_ref
    from actionmesh_b200 import ops

    dev = _cuda()
    c = 3
    x = _feature(h, w, c, 4, dev, torch.Generator(device=dev).manual_seed(oh))
    got = ops.rmbg_upsample(x, h, w, c, torch.empty(oh * ow, c, device=dev), oh, ow).view(oh, ow, c)
    want = rmbg_ref.bilinear_np(x[:, :c].reshape(h, w, c).cpu().numpy(), oh, ow)
    assert np.array_equal(got.cpu().numpy().view(np.int32), want.view(np.int32))
    t = F.interpolate(x[:, :c].reshape(1, h, w, c).permute(0, 3, 1, 2), size=(oh, ow), mode="bilinear",
                      align_corners=False)[0].permute(1, 2, 0)
    mag = F.interpolate(x[:, :c].abs().reshape(1, h, w, c).permute(0, 3, 1, 2), size=(oh, ow), mode="bilinear",
                        align_corners=False)[0].permute(1, 2, 0)
    # torch's CUDA kernel contracts scale * (dst + 0.5) - 0.5 into an FMA, so its source coordinate may differ by an ulp of
    # the coordinate (< in_size): 2 ulp of the blend plus that shift times the largest step between neighbours
    eps = torch.finfo(torch.float32).eps
    step = x[:, :c].abs().max() * 2
    assert ((got - t).abs() <= 2 * eps * mag + eps * max(h, w) * step).all()


@gpu
@pytest.mark.parametrize("h,w", [(1080, 1920), (720, 1280), (512, 512), (480, 640), (300, 457), (1025, 999)])
def test_input_resize_equals_torch_cpu(h, w):
    import rmbg_ref
    from actionmesh_b200 import ops

    dev = _cuda()
    img = np.random.default_rng(h + w).integers(0, 256, (h, w, 3), dtype=np.uint8)
    got = ops.rmbg_resize_input(torch.from_numpy(img).to(dev), torch.empty(1024, 1024, 3, device=dev)).cpu()
    want = rmbg_ref.preprocess(img, (1024, 1024))[0].permute(1, 2, 0)
    if (h, w) in ((1080, 1920), (720, 1280), (512, 512), (480, 640)):
        assert torch.equal(got, want)
    else:
        assert ((got - want).abs() <= 1e-4 * (want + 0.5).abs() + 1e-7).all()  # relative to the resized value / 255


@gpu
def test_mask_head_against_fp64():
    from actionmesh_b200 import ops

    dev = _cuda()
    gen = torch.Generator(device=dev).manual_seed(5)
    h, w = 50, 66
    feat = _feature(h, w, 64, 64, dev, gen).abs()
    wt = torch.randn(577, generator=gen, device=dev) * 0.05
    work = ops.rmbg_mask_head(feat, h, w, wt, (100, 132), (90, 120))
    x = feat[:, :64].double().reshape(1, h, w, 64).permute(0, 3, 1, 2)
    k = wt[:576].double().reshape(3, 3, 64).permute(2, 0, 1)[None]
    ref = F.conv2d(x, k, padding=1)[0, 0] + wt[576].double()
    bound = F.conv2d(x.abs(), k.abs(), padding=1)[0, 0] * 600 * 2.0 ** -24 + abs(wt[576].item()) * 2.0 ** -24
    assert ((work["logits"].double() - ref).abs() <= bound).all()
    soft = torch.sigmoid(F.interpolate(work["logits"][None, None], size=(100, 132), mode="bilinear", align_corners=False))
    assert (work["soft"] - soft[0, 0]).abs().max().item() <= 1e-5   # torch's FMA-contracted source coordinate
    resized = F.interpolate(work["soft"][None, None], size=(90, 120), mode="bilinear", align_corners=False)[0, 0]
    assert (work["resized"] - resized).abs().max().item() <= 1e-5
    r = work["resized"]
    want = ((r - r.min()) / (r.max() - r.min()) * 255).cpu().numpy().astype(np.uint8)
    assert np.array_equal(work["mask"].cpu().numpy(), want)


def _crafted_masks():
    rng = np.random.default_rng(11)
    m = np.zeros((60, 90), np.uint8)
    for k in range(30):
        m[k, k + 50] = 230
    m[10:15, 0:40] = 250
    m[20:26, 0:40] = 240
    m[59, :] = 200
    yield "crafted", m
    yield "constant", np.full((33, 47), 17, np.uint8)
    yield "noise", rng.integers(0, 256, (257, 311), dtype=np.uint8)
    blobs = np.clip(rmbg_ref_smooth(rng, 480, 640), 0, 255).astype(np.uint8)
    yield "blobs", blobs


def rmbg_ref_smooth(rng, h, w):
    x = rng.normal(0, 1, (h // 8 + 2, w // 8 + 2))
    x = np.kron(x, np.ones((8, 8)))[:h, :w]
    return 128 + 90 * x


@gpu
@pytest.mark.parametrize("min_size", [1, 30, 200])
def test_refinement_equals_restatement(min_size):
    import rmbg_ref
    from actionmesh_b200 import ops

    dev = _cuda()
    for name, mask in _crafted_masks():
        rgb = np.random.default_rng(1).integers(0, 256, (*mask.shape, 3), dtype=np.uint8)
        work = {}
        got = ops.rmbg_refine_rgba(torch.from_numpy(rgb).to(dev), torch.from_numpy(mask).to(dev), True, min_size, work=work)
        want = rmbg_ref.refine_rgba_restated(rgb, mask, True, min_size)
        assert int(work["hist"][256]) == rmbg_ref.otsu_cv2(mask)[0], name
        assert np.array_equal(got.cpu().numpy(), want), name
        plain = ops.rmbg_refine_rgba(torch.from_numpy(rgb).to(dev), torch.from_numpy(mask).to(dev), False)
        assert np.array_equal(plain.cpu().numpy(), rmbg_ref.refine_rgba_restated(rgb, mask, False)), name


# ---- the network ----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def remover():
    import rmbg_ref
    from actionmesh_b200.background_removal import B200BackgroundRemover

    dev = _cuda()
    m = B200BackgroundRemover(model_input_size=(1024, 1024)).to(dev)
    m.load_state_dict(rmbg_ref.make_state_dict(0))
    return m


def _weights(size):
    """Seeded weights calibrated at the model input size the test runs (200 x 264: the golden's, from 256 x 320)."""
    import rmbg_ref

    return rmbg_ref.make_state_dict(0) if size != (1024, 1024) else rmbg_ref.make_state_dict(0, size, "cuda")


def _oracle_soft(image, size, tf32: bool):
    import rmbg_ref

    sd = _weights(size)
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = tf32
    try:
        with torch.no_grad():
            soft = rmbg_ref.rmbg_forward(sd, rmbg_ref.preprocess(image, size, "cuda"))
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    return soft[0, 0]


_NETWORK_CASES = [((1024, 1024), (720, 1280)), ((200, 264), (180, 240))]
_network_runs: dict = {}


@pytest.fixture(scope="module", autouse=True)
def _free_network_runs():
    yield
    _network_runs.clear()


def _network_run(size, frame) -> dict:
    """The product and the oracle (cuDNN fp32 and TF32) on one synthetic frame, run once per case."""
    import rmbg_ref
    from actionmesh_b200.background_removal import B200BackgroundRemover

    if (size, frame) not in _network_runs:
        remover = B200BackgroundRemover(model_input_size=size).to(_cuda())
        remover.load_state_dict(_weights(size))
        image = rmbg_ref.synthetic_frame(*frame, 7)
        _, head = remover._run(torch.from_numpy(image).cuda())
        soft, mask = head["soft"].clone(), head["mask"].cpu().numpy()
        fp32 = _oracle_soft(image, size, tf32=False)
        _network_runs[(size, frame)] = dict(remover=remover, image=image, soft=soft, mask=mask, fp32=fp32,
                                            err=(soft - fp32).abs(), err_tf32=(_oracle_soft(image, size, tf32=True) - fp32).abs())
    return _network_runs[(size, frame)]


@gpu
@pytest.mark.parametrize("size,frame", _NETWORK_CASES)
def test_network_ten_times_closer_than_tf32_and_end_to_end(size, frame):
    import rmbg_ref

    r = _network_run(size, frame)
    err, err_tf32 = r["err"], r["err_tf32"]
    print(f"{size}: product max {err.max().item():.3e} mean {err.mean().item():.3e}; "
          f"TF32 oracle max {err_tf32.max().item():.3e} mean {err_tf32.mean().item():.3e}")
    assert err.max().item() * 10 <= err_tf32.max().item() and err.mean().item() * 10 <= err_tf32.mean().item()
    # end to end: the refinement restated on the product's own uint8 mask reproduces its RGBA, and the uint8 soft mask
    # is within 1 of the fp32 oracle's
    image, mask = r["image"], r["mask"]
    rgba = r["remover"].forward(image)
    assert np.array_equal(rgba, rmbg_ref.refine_rgba_restated(image, mask, True, 200))
    want = rmbg_ref.postprocess_mask(r["fp32"][None, None], image.shape[:2])
    diff = np.abs(mask.astype(int) - want.astype(int))
    alpha_ref = rmbg_ref.refine_mask(want, 200)
    print(f"{size}: uint8 mask max diff {diff.max()}, {int((diff > 0).sum())} px differ; binary alpha differs at "
          f"{int((alpha_ref != rgba[..., 3]).sum())} of {alpha_ref.size} px")
    assert diff.max() <= 1


@gpu
@pytest.mark.parametrize("size,frame", [pytest.param(*_NETWORK_CASES[0], marks=pytest.mark.xfail(strict=True, reason=(
    "measured on an H100: max 1.3e-3, mean 1.03e-4 against fp64; the fp32 oracle is 20x closer to fp64, so this is the "
    "three-term split's own error, amplified by the synthetic network at 1024 x 1024 (its TF32 error is 3.5x that at "
    "256 x 320); DESIGN 17"))), _NETWORK_CASES[1]])
def test_network_within_absolute_bounds_of_fp32_oracle(size, frame):
    r = _network_run(size, frame)
    assert r["err"].max().item() <= 1e-3 and r["err"].mean().item() <= 1e-4


@gpu
def test_golden_end_to_end(remover):
    """The reference's own BriaRMBG golden (CPU fp32) at the odd model size: uint8 mask within 1."""
    import rmbg_ref
    from conftest import load_golden

    g = load_golden("rmbg_tiny.pt")
    remover.model_input_size = tuple(g["model_size"])
    image = rmbg_ref.synthetic_frame(*g["frame"], g["frame_seed"])
    _, head = remover._run(torch.from_numpy(image).cuda(), min_size=g["min_size"])
    assert (head["soft"].cpu() - g["soft"]).abs().max().item() <= 1e-3
    assert np.abs(head["mask"].cpu().numpy().astype(int) - g["mask"].numpy().astype(int)).max() <= 1
    remover.model_input_size = (1024, 1024)


@gpu
def test_valid_alpha_passthrough_and_constant_mask(remover):
    from PIL import Image

    from actionmesh_b200 import ops

    rgba = np.zeros((64, 80, 4), np.uint8)
    rgba[..., 3] = 0
    rgba[10:40, 10:50, 3] = 255
    img = Image.fromarray(rgba, "RGBA")
    before = ops.launch_count
    assert remover.process_image(img) is img
    assert ops.launch_count == before
    # ma == mi: all-zero logits weights give a constant soft mask; alpha is then 0 everywhere
    import rmbg_ref

    from actionmesh_b200.background_removal import B200BackgroundRemover

    sd = dict(rmbg_ref.make_state_dict(0))
    sd["side1.weight"] = torch.zeros_like(sd["side1.weight"])
    m = B200BackgroundRemover(model_input_size=(64, 64)).to("cuda")
    m.load_state_dict(sd)
    out = m.process_image(Image.fromarray(rgba[..., :3], "RGB"))
    arr = np.asarray(out)
    assert out.mode == "RGBA" and (arr[..., 3] == 0).all() and np.array_equal(arr[..., :3], rgba[..., :3])
    # an RGBA frame whose alpha is not valid goes through the network (converted to RGB first)
    thin = rgba.copy()
    thin[..., 3] = 255
    res = m.process_images([Image.fromarray(thin, "RGBA")])
    assert len(res) == 1 and res[0].mode == "RGBA" and (np.asarray(res[0])[..., 3] == 0).all()


@gpu
def test_pipeline_uses_remover_before_preprocessor(remover):
    """ActionMeshB200Pipeline's background_removal seam, built with tiny dimensions: the call completes, and the frames
    reaching Stage 0 are the remover's process_images followed by the preprocessor's, called directly."""
    from PIL import Image

    import rmbg_ref
    from actionmesh_b200.autoencoder import AutoencoderConfig, B200Autoencoder
    from actionmesh_b200.denoiser import B200Denoiser, DenoiserConfig
    from actionmesh_b200.image_encoder import B200ImageEncoder
    from actionmesh_b200.pipeline import ActionMeshB200Pipeline, ActionMeshInput
    from actionmesh_b200.preprocess import B200FramePreprocessor
    from oracle import autoencoder_oracle as ao
    from oracle import synth

    n_frames, N, V = 17, 31, 200
    enc = B200ImageEncoder(hidden_size=256, num_layers=2, num_heads=4).to("cuda")
    enc.init_random_(seed=5)
    dcfg = DenoiserConfig(num_layers=3, num_attention_heads=2, width=256, cross_attention_dim=256, in_channels=64,
                          inflated_layers=(0, 1, 2))
    den = B200Denoiser(dcfg).to("cuda")
    den.load_state_dict(synth.make_state_dict(dcfg, 17))
    ae = B200Autoencoder(AutoencoderConfig(width=256, num_layers=2, num_attention_heads=2, temporal_context_size=16)).to("cuda")
    ae.load_state_dict(ao.make_autoencoder_state_dict(ao.AutoencoderConfig(width=256, num_layers=2, num_attention_heads=2), 99))
    g = torch.Generator().manual_seed(3)
    pts = torch.randn(V, 3, generator=g)
    pts = pts / pts.norm(dim=-1, keepdim=True) * 0.5

    class AnchorMesh:
        vertices, vertex_normals = pts.numpy(), torch.nn.functional.normalize(pts, dim=-1).numpy()
        faces = torch.randint(0, V, (300, 3), generator=g).numpy()

    anchor_latent = torch.randn(1, N, 64, generator=g)
    seen = {}

    def stage0(image, generator, num_inference_steps, guidance_scale):
        seen["image"] = image
        return anchor_latent, AnchorMesh

    class Recording(B200FramePreprocessor):
        def process_images(self, images):
            seen["frames"] = super().process_images(images)
            return seen["frames"]

    remover.model_input_size = (128, 128)
    frames = [Image.fromarray(rmbg_ref.synthetic_frame(96, 112, s), "RGB") for s in range(n_frames)]
    want = B200FramePreprocessor().process_images(remover.process_images(list(frames)))
    pipe = ActionMeshB200Pipeline("actionmesh_b200.yaml", image_to_3d=stage0, background_removal=remover,
                                  image_process=Recording(),
                                  config_updates={"model.temporal_3D_denoiser.num_tokens_nominal": N, "stage_1_steps": 2})
    pipe.image_encoder, pipe.temporal_3D_denoiser, pipe.temporal_3D_vae = enc, den, ae
    pipe.to("cuda")
    meshes = pipe(ActionMeshInput(list(frames), torch.arange(n_frames, dtype=torch.float32)), seed=44, stage_0_steps=2,
                  guidance_scales=[3.0])
    remover.model_input_size = (1024, 1024)
    assert len(meshes) == n_frames and all(np.isfinite(m.vertices).all() for m in meshes)
    assert len(seen["frames"]) == len(want)
    for a, b in zip(seen["frames"], want):
        assert np.array_equal(np.asarray(a), np.asarray(b))
    assert np.array_equal(np.asarray(seen["image"]), np.asarray(want[0]))
