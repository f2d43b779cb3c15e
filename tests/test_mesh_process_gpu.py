"""Anchor-mesh post-processing on the GPU (-m gpu): the decimation and floater kernels against the numpy restatement bit for
bit, determinism, full-size decimation of depth-9 Stage 0 meshes to 40 000 faces, and B200MeshPostprocessor selected in
ActionMeshB200Pipeline through `_target_`."""
import json
import os
import tempfile

import numpy as np
import pytest
import torch

import mesh_process_ref as ref
import triposg_vae_ref as tref
from actionmesh_b200.mesh_input import clean_topology

pytestmark = pytest.mark.gpu


def _gpu(v, f, target=None, threshold=None):
    from actionmesh_b200 import ops
    from actionmesh_b200.mesh_process import decimate, remove_floaters

    pos = torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64)).cuda()
    ft = torch.from_numpy(np.ascontiguousarray(f, dtype=np.int32)).cuda()
    work, scan = ops.mesh_scan_scratch(len(v), len(f), "cuda")
    rounds = 0
    if target is not None:
        pos, ft, rounds = decimate(pos, ft, target, work, scan)
    if threshold is not None:
        pos, ft = remove_floaters(pos, ft, threshold, work, scan)
    return pos.cpu().numpy(), ft.cpu().numpy().astype(np.int64), rounds


def _dmc_mesh(name):
    field = tref.sphere if name == "sphere" else tref.torus
    v, f = tref.dmc_numpy(tref.dense_grid(field, 97))
    return clean_topology(v.astype(np.float64), f.astype(np.int64))


def _same(a, b):
    """Bit-identical float64 arrays (and equal shapes)."""
    return a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64))


def _check_decimation(v, f, target):
    rv, rf, rrounds = ref.decimate(v, f, target)
    gv, gf, grounds = _gpu(v, f, target)
    assert grounds == rrounds
    assert np.array_equal(gf, rf)
    assert _same(gv, rv), float(np.abs(gv - rv).max()) if gv.shape == rv.shape else (gv.shape, rv.shape)
    gv2, gf2, _ = _gpu(v, f, target)                                     # two runs are identical
    assert _same(gv2, gv) and np.array_equal(gf2, gf)
    return gv, gf


@pytest.mark.parametrize("target", [4000, 1000])
@pytest.mark.parametrize("name", ["sphere", "torus"])
def test_decimation_matches_restatement_on_closed_surfaces(amb_lib, name, target):
    v, f = _dmc_mesh(name)
    gv, gf = _check_decimation(v, f, target)
    closed, chi, _ = tref.mesh_stats(gv, gf)
    assert len(gf) in (target - 1, target) and closed and chi == (2 if name == "sphere" else 0)


def test_decimation_matches_restatement_on_open_grid(amb_lib):
    v, f = ref.grid_mesh(24)
    gv, gf = _check_decimation(v, f, 200)
    assert len(gf) in (199, 200) and np.all(gv[:, 2] == 0.0)


def test_decimation_matches_restatement_on_nonmanifold_soup(amb_lib):
    v, f = ref.soup_mesh()
    _check_decimation(v, f, 100)


def test_decimation_matches_restatement_on_1000_face_fan(amb_lib):
    v, f = ref.fan_mesh(1000)
    gv, gf = _check_decimation(v, f, 100)
    assert len(gf) in (99, 100)


def test_floater_mesh_matches_restatement(amb_lib):
    v, f = ref.floater_mesh()
    _check_decimation(v, f, 800)
    for thr in (0.005, 0.02, 0.2):
        rv, rf = ref.remove_floaters(v, f, thr)
        gv, gf, _ = _gpu(v, f, threshold=thr)
        assert np.array_equal(gf, rf) and _same(gv, rv)
    gv, gf, _ = _gpu(v, f, threshold=2.0)                                # nothing kept: unchanged
    assert np.array_equal(gf, f) and _same(gv, v)
    rv, rf, _ = ref.decimate(v, f, 800)
    rv, rf = ref.remove_floaters(rv, rf, 0.02)
    gv, gf, _ = _gpu(v, f, target=800, threshold=0.02)
    assert np.array_equal(gf, rf) and _same(gv, rv)


@pytest.mark.parametrize("name", ["sphere", "torus"])
def test_full_size_depth9_decimation_to_40000(amb_lib, name):
    from actionmesh_b200.evaluation import compute_chamfer_score
    from actionmesh_b200.mesh_process import B200MeshPostprocessor
    from actionmesh_b200.triposg_vae import make_mesh, mesh_from_grid, refine_octree

    field = tref.sphere if name == "sphere" else tref.torus
    v, f = mesh_from_grid(refine_octree(field, tref.BOUNDS, 9), tref.BOUNDS, 9)
    mesh = make_mesh(v, f)
    v0, f0 = clean_topology(v.astype(np.float64), f.astype(np.int64))
    assert len(f0) > 800_000
    _, chi0, vol0 = tref.mesh_stats(v0, f0)
    out = B200MeshPostprocessor(face_decimation=40000, verbose=False).process_mesh(mesh)
    assert np.array_equal(mesh.faces, f) and np.array_equal(mesh.vertices, v)                # input untouched
    dv, df = np.asarray(out.vertices), np.asarray(out.faces)
    closed, chi, vol = tref.mesh_stats(dv, df)
    voxel = 2.01 / 512
    dist = ref.point_mesh_distance(dv, v0, f0)
    # vertex-to-vertex Chamfer against the dense input: about half the decimated mesh's mean edge length by construction
    chamfer = compute_chamfer_score(dv, v0)
    e = np.concatenate([df[:, [0, 1]], df[:, [1, 2]], df[:, [2, 0]]])
    edge = float(np.linalg.norm(dv[e[:, 0]] - dv[e[:, 1]], axis=1).mean())
    report = {"mesh": name, "faces_in": len(f0), "faces_out": len(df), "vertices_out": len(dv), "chi": chi,
              "volume_ratio": vol / vol0, "max_dist_voxels": float(dist.max() / voxel), "chamfer": chamfer,
              "mean_edge": edge, "voxel": voxel}
    with open(os.path.join(tempfile.gettempdir(), f"mesh_process_{name}_depth9.json"), "w") as fh:
        json.dump(report, fh)
    print("depth-9 decimation:", report)
    assert len(df) in (39999, 40000) and closed and chi == chi0
    assert abs(vol / vol0 - 1) < 0.01
    assert dist.max() <= 0.5 * voxel
    assert chamfer <= 0.6 * edge


def test_pipeline_selects_postprocessor_through_target(amb_lib):
    """ActionMeshB200Pipeline with `model.mesh_process._target_` pointing at B200MeshPostprocessor and face_decimation=2000:
    every output mesh has the post-processed anchor's faces and frame 0 its vertices."""
    from PIL import Image

    from actionmesh_b200.autoencoder import AutoencoderConfig, B200Autoencoder
    from actionmesh_b200.denoiser import B200Denoiser, DenoiserConfig
    from actionmesh_b200.image_encoder import B200ImageEncoder
    from actionmesh_b200.mesh_process import B200MeshPostprocessor
    from actionmesh_b200.pipeline import ActionMeshB200Pipeline, ActionMeshInput
    from actionmesh_b200.triposg_vae import make_mesh
    from oracle import autoencoder_oracle as ao
    from oracle import synth

    N, n_frames = 31, 16
    enc = B200ImageEncoder(hidden_size=256, num_layers=2, num_heads=4).to("cuda")
    enc.init_random_(seed=5)
    dcfg = DenoiserConfig(num_layers=3, num_attention_heads=2, width=256, cross_attention_dim=256, in_channels=64,
                          inflated_layers=(0, 1, 2))
    den = B200Denoiser(dcfg).to("cuda")
    den.load_state_dict(synth.make_state_dict(dcfg, 17))
    ae = B200Autoencoder(AutoencoderConfig(width=256, num_layers=2, num_attention_heads=2, temporal_context_size=16)).to("cuda")
    ae.load_state_dict(ao.make_autoencoder_state_dict(ao.AutoencoderConfig(width=256, num_layers=2, num_attention_heads=2), 99))

    v, f = tref.dmc_numpy(tref.dense_grid(tref.sphere, 97))
    v = (v / 48.0 - 1.0).astype(np.float32)                            # grid units -> [-1, 1]
    anchor = make_mesh(v, f.astype(np.int64))

    def image_to_3d(image, generator, num_inference_steps, guidance_scale):
        return torch.randn(1, N, 64, generator=torch.Generator().manual_seed(1)), anchor

    rng = np.random.default_rng(7)
    frames = [Image.fromarray(rng.integers(0, 255, (96, 96, 3), dtype=np.uint8), "RGB") for _ in range(n_frames)]
    pipe = ActionMeshB200Pipeline("actionmesh_b200.yaml", image_to_3d=image_to_3d,
                                  config_updates={"model.temporal_3D_denoiser.num_tokens_nominal": N, "stage_1_steps": 2,
                                                  "model.mesh_process._target_": "actionmesh_b200.mesh_process.B200MeshPostprocessor"})
    assert isinstance(pipe.mesh_process, B200MeshPostprocessor)
    pipe.image_encoder, pipe.temporal_3D_denoiser, pipe.temporal_3D_vae = enc, den, ae
    pipe.to("cuda")
    meshes = pipe(ActionMeshInput(frames, torch.arange(n_frames, dtype=torch.float32)), seed=44, stage_0_steps=2,
                  face_decimation=2000, guidance_scales=[3.0])
    expected = B200MeshPostprocessor(face_decimation=2000, floaters_threshold=0.02).process_mesh(anchor)
    assert len(expected.faces) in (1999, 2000) and len(meshes) == n_frames
    assert all(np.array_equal(m.faces, expected.faces) for m in meshes)
    assert np.array_equal(meshes[0].vertices, np.asarray(expected.vertices, dtype=np.float32))
    assert all(np.isfinite(m.vertices).all() for m in meshes)
