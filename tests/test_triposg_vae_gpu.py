"""Stage 0's anchor mesh on the GPU (-m gpu): B200TripoSGVAE.decode against the reference's TripoSG VAE (golden) and the fp32
restatement at full width, the octree refinement against the reference's flash_extract_geometry with analytic fields, the
dual-marching-cubes kernel against its numpy restatement, and TripoSGStage0 -> ActionMeshB200Pipeline end to end."""
import json
import os
import tempfile

import numpy as np
import pytest
import torch

import triposg_vae_ref as ref
from conftest import load_golden

pytestmark = pytest.mark.gpu


def _vae(width, heads, layers, seed):
    from actionmesh_b200.triposg_vae import B200TripoSGVAE

    sd = ref.make_state_dict(width, heads, layers, seed=seed)
    vae = B200TripoSGVAE(width_decoder=width, num_attention_heads=heads, num_layers_decoder=layers).to("cuda")
    vae.load_state_dict(sd)
    return vae, sd


def test_decode_matches_reference_tiny(amb_lib):
    g = load_golden("triposg_vae_tiny.pt")
    c = g["config"]
    vae, _ = _vae(c["width_decoder"], c["num_attention_heads"], c["num_layers_decoder"], g["seed"])
    out = vae.decode(g["z"].cuda(), g["points"].cuda())
    assert out.shape == (1, 4096, 1) and out.dtype == torch.float32
    err = float((out.cpu() - g["logits"]).norm() / g["logits"].norm())
    assert err <= 2e-2, err
    # chunked query path gives the same logits as one pass
    ctx = vae.prepare(g["z"][0].cuda())
    a = vae.query(ctx, g["points"][0].cuda())
    b = vae.query(ctx, g["points"][0].cuda(), chunk=1000)
    assert torch.equal(a, b) and torch.equal(a[:, :1], out[0])


def test_decode_full_width_matches_fp32_restatement(amb_lib):
    vae, sd = _vae(1024, 8, 16, seed=77)
    g = torch.Generator().manual_seed(3)
    z = torch.randn(1, 2048, 64, generator=g).cuda()
    pts = (torch.rand(1, 65536, 3, generator=g) * 2.01 - 1.005).cuda()
    out = vae.decode(z, pts)
    refl = ref.decode_fp32(sd, z, pts, 8, 16)
    err = float((out - refl).norm() / refl.norm())
    print(f"full-width decode rel err {err:.3e}")
    assert err <= 2e-2, err


@pytest.mark.parametrize("name", ["sphere", "torus"])
@pytest.mark.parametrize("depth", [7, 8])
def test_octree_refinement_matches_reference(amb_lib, name, depth):
    from actionmesh_b200.triposg_vae import refine_octree

    gold = load_golden("triposg_vae_tiny.pt")["fields"][(name, depth)]
    field = ref.sphere if name == "sphere" else ref.torus
    grid = refine_octree(field, ref.BOUNDS, depth).reshape(-1)
    assert grid.shape[0] == gold["side"] ** 3
    idx = torch.nonzero(torch.isfinite(grid)).reshape(-1).to(torch.int32)
    val = grid[idx.long()]
    assert idx.numel() == gold["count"]
    assert torch.equal(idx[:2000].cpu(), gold["head_index"]) and torch.equal(val[:2000].cpu(), gold["head_values"])
    assert ref.sha256(idx) == gold["sha256_index"]
    assert ref.sha256(val) == gold["sha256_values"]


def _check_dmc(grid_np):
    from actionmesh_b200 import ops

    grid = torch.from_numpy(grid_np).cuda()
    v1, f1 = ops.dual_marching_cubes(grid)
    v2, f2 = ops.dual_marching_cubes(grid)
    assert torch.equal(v1, v2) and torch.equal(f1, f2)          # deterministic
    rv, rf = ref.dmc_numpy(grid_np)
    assert np.array_equal(f1.cpu().numpy().astype(np.int64), rf)
    assert np.array_equal(v1.cpu().numpy().view(np.int32), rv.view(np.int32))   # bit for bit
    return v1.cpu().numpy(), f1.cpu().numpy()


@pytest.mark.parametrize("name", ["sphere", "torus"])
def test_dmc_kernel_matches_restatement(amb_lib, name):
    field = ref.sphere if name == "sphere" else ref.torus
    v, f = _check_dmc(ref.dense_grid(field, 97))
    closed, chi, vol = ref.mesh_stats(v, f)
    assert closed and chi == (2 if name == "sphere" else 0) and vol > 0


@pytest.mark.parametrize("name", ["sphere", "torus"])
def test_dmc_kernel_on_refined_band_with_nan(amb_lib, name):
    from actionmesh_b200.triposg_vae import mesh_from_grid, refine_octree

    field = ref.sphere if name == "sphere" else ref.torus
    grid = refine_octree(field, ref.BOUNDS, 8)
    assert torch.isnan(grid).any()
    v, f = _check_dmc(grid.cpu().numpy())
    closed, chi, vol = ref.mesh_stats(v, f)
    assert closed and chi == (2 if name == "sphere" else 0) and vol > 0
    mv, mf = mesh_from_grid(grid, ref.BOUNDS, 8)
    assert mv.dtype == np.float32 and np.array_equal(mf, f.astype(np.int64))
    # the reference's scale: / 2**depth (not the 252 cells the grid spans) * bbox size + bbox min
    assert np.allclose(mv, (v / 256.0 * 2.01 - 1.005).astype(np.float32), atol=1e-6)


def test_stage0_mesh_extractor_end_to_end(amb_lib):
    """TripoSGStage0 (tiny DiT) + B200TripoSGVAE.extract_mesh (tiny VAE, octree depth 7) -> a mesh carried through Stage II of
    ActionMeshB200Pipeline; its Chamfer distance to the mesh the same extractor builds from the fp32 restatement's logits."""
    from PIL import Image

    from actionmesh_b200.autoencoder import AutoencoderConfig, B200Autoencoder
    from actionmesh_b200.denoiser import B200Denoiser, DenoiserConfig
    from actionmesh_b200.evaluation import compute_chamfer_score
    from actionmesh_b200.image_encoder import B200ImageEncoder
    from actionmesh_b200.pipeline import ActionMeshB200Pipeline, ActionMeshInput
    from actionmesh_b200.stage0 import B200TripoSGDiT, TripoSGStage0
    from actionmesh_b200.triposg_vae import B200TripoSGVAE, mesh_from_grid, refine_octree
    from oracle import autoencoder_oracle as ao
    from oracle import synth

    class _TinyCfg:
        in_channels, num_layers, num_attention_heads, width, mlp_ratio, cross_attention_dim = 64, 5, 2, 256, 4.0, 128

    depth = 7
    dit = B200TripoSGDiT(num_attention_heads=2, width=256, in_channels=64, num_layers=5, cross_attention_dim=128).to("cuda")
    dit.load_state_dict(synth.make_state_dict(_TinyCfg(), 4242))
    sd = ref.make_state_dict(256, 2, 2, seed=8)
    g = torch.Generator().manual_seed(12)
    emb = torch.randn(1, 9, 128, generator=g).cuda()
    vae = B200TripoSGVAE(width_decoder=256, num_attention_heads=2, num_layers_decoder=2).to("cuda")
    vae.load_state_dict(sd)
    stage0 = TripoSGStage0(dit, image_encoder=None, mesh_extractor=lambda lat: vae.extract_mesh(lat, octree_depth=depth),
                           shift=3.0, num_tokens=64)
    # centre the random decoder's field: shift proj_out's bias so that half of the coarse grid is inside
    lat = stage0.denoise(emb, torch.randn(1, 64, 64, generator=torch.Generator().manual_seed(7)).cuda(), 2, 2.0)
    a = torch.linspace(-1.005, 1.005, 64)
    xyz = torch.stack(torch.meshgrid(a, a, a, indexing="ij"), -1).reshape(1, -1, 3).cuda()
    sd["decoder.proj_out.bias"] = sd["decoder.proj_out.bias"] + ref.decode_fp32(sd, lat, xyz, 2, 2).median().cpu()
    vae.load_state_dict(sd)

    latent, mesh = stage0(emb, generator=torch.Generator().manual_seed(7), num_inference_steps=2, guidance_scale=2.0)
    assert torch.equal(latent, lat)
    assert len(mesh.faces) > 100 and mesh.vertex_normals.shape == mesh.vertices.shape
    assert np.isfinite(mesh.vertices).all()

    _, kv = ref.decode_fp32(sd, lat, xyz[:, :1], 2, 2, return_kv=True)
    grid32 = refine_octree(lambda p: ref.decode_fp32(sd, lat, p[None], 2, 2, kv_cache=kv)[0], ref.BOUNDS, depth)
    v32, _ = mesh_from_grid(grid32, ref.BOUNDS, depth)
    chamfer = compute_chamfer_score(mesh.vertices, v32)
    voxel = 2.01 / 126
    report = {"chamfer": chamfer, "voxel": voxel, "vertices": len(mesh.vertices), "faces": len(mesh.faces)}
    with open(os.path.join(tempfile.gettempdir(), "triposg_vae_chamfer.json"), "w") as fh:
        json.dump(report, fh)
    print("stage0 mesh chamfer vs fp32 restatement:", report)
    assert chamfer <= voxel, report

    # ... carried through Stage II of the pipeline (tiny Stage-I / Stage-II models, as tests/test_pipeline_gpu.py)
    N = 31
    enc = B200ImageEncoder(hidden_size=256, num_layers=2, num_heads=4).to("cuda")
    enc.init_random_(seed=5)
    dcfg = DenoiserConfig(num_layers=3, num_attention_heads=2, width=256, cross_attention_dim=256, in_channels=64,
                          inflated_layers=(0, 1, 2))
    den = B200Denoiser(dcfg).to("cuda")
    den.load_state_dict(synth.make_state_dict(dcfg, 17))
    ae = B200Autoencoder(AutoencoderConfig(width=256, num_layers=2, num_attention_heads=2, temporal_context_size=16)).to("cuda")
    ae.load_state_dict(ao.make_autoencoder_state_dict(ao.AutoencoderConfig(width=256, num_layers=2, num_attention_heads=2), 99))

    anchor = {}

    def image_to_3d(image, generator, num_inference_steps, guidance_scale):
        _, m = stage0(emb, generator=generator, num_inference_steps=num_inference_steps, guidance_scale=guidance_scale)
        anchor["mesh"] = m
        return torch.randn(1, N, 64, generator=torch.Generator().manual_seed(1)), m

    n_frames = 16
    rng = np.random.default_rng(7)
    frames = [Image.fromarray(rng.integers(0, 255, (96, 96, 3), dtype=np.uint8), "RGB") for _ in range(n_frames)]
    pipe = ActionMeshB200Pipeline("actionmesh_b200.yaml", image_to_3d=image_to_3d,
                                  config_updates={"model.temporal_3D_denoiser.num_tokens_nominal": N, "stage_1_steps": 2})
    pipe.image_encoder, pipe.temporal_3D_denoiser, pipe.temporal_3D_vae = enc, den, ae
    pipe.to("cuda")
    meshes = pipe(ActionMeshInput(frames, torch.arange(n_frames, dtype=torch.float32)), seed=44, stage_0_steps=2,
                  guidance_scales=[3.0])
    assert len(meshes) == n_frames
    am = anchor["mesh"]                                  # the pipeline seeds Stage 0 itself: its own anchor mesh
    assert len(am.faces) > 100 and all(m.vertices.shape == am.vertices.shape and np.isfinite(m.vertices).all() for m in meshes)
    assert np.array_equal(meshes[0].faces, am.faces) and np.array_equal(meshes[0].vertices, am.vertices)
