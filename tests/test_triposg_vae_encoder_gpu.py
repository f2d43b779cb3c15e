"""The mesh-input path on the GPU (-m gpu): the farthest-point-sampling kernel against its numpy restatement, the TripoSG VAE
encoder against the reference (golden) and the fp32 restatement at full width, and ActionMeshB200PipelineWithMeshInput end
to end."""
import numpy as np
import pytest
import torch

import triposg_vae_encoder_ref as ref
import triposg_vae_ref as dref
from conftest import load_golden

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("N", [1000, 8192, 16384])
@pytest.mark.parametrize("K", [1, 256, 2048])
def test_fps_kernel_equals_restatement(amb_lib, B, N, K):
    from actionmesh_b200 import ops

    g = torch.Generator().manual_seed(N + K + B)
    surface = torch.randn(B, N, 6, generator=g)          # xyz read in place from 6-channel rows
    start = torch.randint(high=N, size=(B,), generator=g)
    start[0] = N - 1
    got = ops.farthest_point_sample(surface.cuda(), K, start)
    assert got.shape == (B, K) and got.dtype == torch.int64
    for b in range(B):
        want = ref.fps_numpy(surface[b, :, :3].numpy(), K, int(start[b]))
        assert np.array_equal(got[b].cpu().numpy(), want), b
    # device-side start indices give the same result, and the kernel is deterministic
    assert torch.equal(ops.farthest_point_sample(surface.cuda(), K, start.cuda()), got)


def test_fps_kernel_ties_duplicates_and_exhaustion(amb_lib):
    from actionmesh_b200 import ops

    g = torch.Generator().manual_seed(5)
    base = torch.randint(-3, 4, (37, 3), generator=g).float()              # an integer lattice: many equal distances
    pts = base[torch.randint(0, 37, (3001,), generator=g)]                 # every point duplicated many times
    for start, K in ((0, 64), (3000, 64), (17, 3001)):
        got = ops.farthest_point_sample(pts[None].cuda(), K, torch.tensor([start]))[0].cpu().numpy()
        assert np.array_equal(got, ref.fps_numpy(pts.numpy(), K, start)), (start, K)
    assert got[-1] == 0                                                     # exhausted: argmax repeats the lowest index


def test_fps_rejects_large_clouds(amb_lib):
    from actionmesh_b200 import AmbError, ops

    with pytest.raises(AmbError, match="points"):
        ops.farthest_point_sample(torch.zeros(1, 16385, 3, device="cuda"), 16, torch.tensor([0]))
    with pytest.raises(AmbError, match="start"):
        ops.farthest_point_sample(torch.zeros(1, 100, 3, device="cuda"), 16, torch.tensor([100]))


def _vae(c, sd_enc, decoder_seed=1):
    from actionmesh_b200.triposg_vae import B200TripoSGVAE

    sd = dref.make_state_dict(c["width_decoder"], c["num_attention_heads"], c["num_layers_decoder"], seed=decoder_seed)
    sd.update(sd_enc)
    vae = B200TripoSGVAE(width_encoder=c["width_encoder"], num_layers_encoder=c["num_layers_encoder"],
                         width_decoder=c["width_decoder"], num_layers_decoder=c["num_layers_decoder"],
                         num_attention_heads=c["num_attention_heads"]).to("cuda")
    vae.load_state_dict(sd)
    return vae


def _rel(a, b):
    return float((a.float().cpu() - b.float().cpu()).norm() / b.float().cpu().norm())


def test_tiny_encoder_matches_reference(amb_lib):
    g = load_golden("triposg_vae_encoder_tiny.pt")
    c = g["config"]
    sd = ref.make_encoder_state_dict(c["width_encoder"], c["num_attention_heads"], c["num_layers_encoder"], seed=g["seed"])
    vae = _vae(c, sd)
    from actionmesh_b200 import ops

    surface = g["surface"].cuda()
    n, m = surface.shape[1], 4 * g["num_tokens"]
    assert np.array_equal(np.random.default_rng(g["subset_seed"]).choice(n, m, replace=m > n), g["subset"].numpy())
    selected = surface[:, g["subset"].cuda()]
    idx = ops.farthest_point_sample(selected, g["num_tokens"], torch.tensor([g["fps_start"]]))
    assert torch.equal(idx[0].cpu(), g["fps_index"])
    sampled = selected[:, idx[0]]
    quant = vae.encode_points(surface[0], sampled[0])
    mean, logvar = g["quant"][0].chunk(2, dim=-1)
    from actionmesh_b200.triposg_vae import DiagonalGaussianDistribution

    post = DiagonalGaussianDistribution(quant[None])
    e_mean, e_logvar = _rel(post.mean, mean[None]), _rel(post.logvar, logvar.clamp(-30, 20)[None])
    z = post.sample(eps=g["eps"])
    e_z = _rel(z, g["latent"])
    print(f"tiny encoder rel err: mean {e_mean:.2e} logvar {e_logvar:.2e} latent {e_z:.2e}")
    assert e_mean <= 2e-2 and e_logvar <= 2e-2 and e_z <= 2e-2, (e_mean, e_logvar, e_z)
    assert torch.allclose(post.std, torch.exp(0.5 * post.logvar), rtol=1e-6)


def test_full_width_encoder_matches_fp32_restatement(amb_lib):
    c = dict(width_encoder=512, num_attention_heads=8, num_layers_encoder=8, width_decoder=1024, num_layers_decoder=1)
    sd = ref.make_encoder_state_dict(512, 8, 8, seed=31)
    vae = _vae(c, sd)
    surface = ref.sphere_surface(16384, 4).cuda()
    sampled, _ = vae.sample_features(surface, 2048, seed=3, generator=torch.Generator().manual_seed(3))
    out = vae.encode_points(surface[0], sampled[0])
    want = ref.encode_fp32(sd, surface, sampled, 8, 8)[0]
    err = _rel(out, want)
    print(f"full-width encoder rel err {err:.3e}")
    assert out.shape == (2048, 128) and err <= 2e-2, err


def test_encode_to_latent_is_reproducible(amb_lib):
    g = load_golden("triposg_vae_encoder_tiny.pt")
    c = g["config"]
    vae = _vae(c, ref.make_encoder_state_dict(c["width_encoder"], c["num_attention_heads"], c["num_layers_encoder"], seed=2))
    surface = ref.sphere_surface(16384, 6).cuda()
    a = vae.encode_to_latent(surface, seed=44, generator=torch.Generator().manual_seed(44))
    b = vae.encode_to_latent(surface, seed=44, generator=torch.Generator().manual_seed(44))
    assert a.shape == (1, 2048, 64) and a.dtype == torch.float32 and torch.isfinite(a).all()
    assert torch.equal(a, b)
    gen = torch.Generator().manual_seed(44)
    post = vae.encode(surface, seed=44, generator=gen).latent_dist         # the same draws through the public pieces
    assert post.mean.shape == post.logvar.shape == post.std.shape == (1, 2048, 64)
    assert torch.equal(post.sample(gen), a)


def test_random_init_keeps_decoder_weights(amb_lib):
    from actionmesh_b200.triposg_vae import B200TripoSGVAE

    a = B200TripoSGVAE(width_decoder=256, num_attention_heads=2, num_layers_decoder=2).to("cuda")   # no encoder (head_dim 256)
    a.init_random_(seed=9)
    b = B200TripoSGVAE(width_decoder=256, num_attention_heads=2, num_layers_decoder=2, width_encoder=256).to("cuda")
    b.init_random_(seed=9)
    assert not a._has_encoder and b._has_encoder
    for k, v in a._w.items():
        assert torch.equal(v, b._w[k]), k


def _split_seam_mesh(n_lat=12, n_lon=16, radii=(0.9, 0.6, 0.45), offset=(2.0, -1.0, 0.5)):
    """A UV sphere (ellipsoid) whose every quad owns its four corners: a mesh of seams, 4 vertices per quad."""
    th = np.linspace(0.0, np.pi, n_lat + 1)
    ph = np.linspace(0.0, 2 * np.pi, n_lon + 1)
    grid = np.stack([np.sin(th)[:, None] * np.cos(ph)[None], np.sin(th)[:, None] * np.sin(ph)[None],
                     np.cos(th)[:, None] * np.ones_like(ph)[None]], axis=-1) * np.array(radii) + np.array(offset)
    verts, faces = [], []
    for i in range(n_lat):
        for j in range(n_lon):
            b = len(verts)
            verts.extend([grid[i, j], grid[i + 1, j], grid[i + 1, j + 1], grid[i, j + 1]])
            faces.extend([(b, b + 1, b + 2), (b, b + 2, b + 3)])
    return np.array(verts), np.array(faces, dtype=np.int64)


def test_mesh_input_pipeline_end_to_end(amb_lib):
    from PIL import Image

    from actionmesh_b200.autoencoder import AutoencoderConfig, B200Autoencoder
    from actionmesh_b200.denoiser import B200Denoiser, DenoiserConfig
    from actionmesh_b200.image_encoder import B200ImageEncoder
    from actionmesh_b200.pipeline import ActionMeshB200PipelineWithMeshInput, ActionMeshInput, Mesh
    from oracle import autoencoder_oracle as ao
    from oracle import synth

    N, n_frames = 2048, 16
    c = dict(width_encoder=256, num_attention_heads=4, num_layers_encoder=2, width_decoder=512, num_layers_decoder=1)
    vae = _vae(c, ref.make_encoder_state_dict(256, 4, 2, seed=12))
    enc = B200ImageEncoder(hidden_size=256, num_layers=2, num_heads=4).to("cuda")
    enc.init_random_(seed=5)
    dcfg = DenoiserConfig(num_layers=3, num_attention_heads=2, width=256, cross_attention_dim=256, in_channels=64,
                          inflated_layers=(0, 1, 2))
    den = B200Denoiser(dcfg).to("cuda")
    den.load_state_dict(synth.make_state_dict(dcfg, 17))
    ae = B200Autoencoder(AutoencoderConfig(width=256, num_layers=2, num_attention_heads=2, temporal_context_size=16)).to("cuda")
    ae.load_state_dict(ao.make_autoencoder_state_dict(ao.AutoencoderConfig(width=256, num_layers=2, num_attention_heads=2), 99))
    pipe = ActionMeshB200PipelineWithMeshInput("actionmesh_b200.yaml",
                                               config_updates={"model.temporal_3D_denoiser.num_tokens_nominal": N,
                                                               "stage_1_steps": 2})
    pipe.image_encoder, pipe.temporal_3D_denoiser, pipe.temporal_3D_vae, pipe.vae = enc, den, ae, vae
    pipe.to("cuda")
    v, f = _split_seam_mesh()
    rng = np.random.default_rng(7)
    frames = [Image.fromarray(rng.integers(0, 255, (96, 96, 3), dtype=np.uint8), "RGB") for _ in range(n_frames)]
    ts = torch.arange(n_frames, dtype=torch.float32)

    def run():
        return pipe(ActionMeshInput(list(frames), ts.clone()), Mesh(vertices=v.copy(), faces=f.copy()), seed=44,
                    guidance_scales=[3.0])

    meshes = run()
    assert len(meshes) == n_frames
    for m in meshes:
        assert np.asarray(m.vertices).shape == v.shape and np.array_equal(np.asarray(m.faces), f)
        assert np.isfinite(m.vertices).all()
    scale = (v.max(axis=0) - v.min(axis=0)).max()
    err = np.abs(np.asarray(meshes[0].vertices) - v).max()
    assert err <= 4 * np.finfo(np.float32).eps * scale * 2, err         # fp32 round-off of normalize -> denormalize
    assert np.abs(np.asarray(meshes[-1].vertices) - v).max() > 0       # later frames move
    again = run()
    assert all(np.array_equal(a.vertices, b.vertices) for a, b in zip(meshes, again))
