"""The command line's whole path on the GPU (-m gpu): frames on disk -> `run_actionmesh` -> the files on disk, on the tiny
checkpoint tree of tests/standalone_tree.py.  The files hold what run_actionmesh returned, and that is what the same pipeline
returns when called directly."""
import io
import os

import numpy as np
import pytest
import torch

import glb_check
import standalone_tree as st

pytestmark = pytest.mark.gpu

UPDATES = {"model.temporal_3D_denoiser.num_tokens_nominal": st.N_TOKENS, "stage_0_steps": 2, "stage_1_steps": 2}


@pytest.fixture(scope="module")
def root(tmp_path_factory, amb_lib):
    """The checkpoint tree, its VAE's field centred on the anchor latents of seeds 44 and 45 so that Stage 0 yields a
    surface (the recipe of test_standalone_pipeline_gpu.py)."""
    from actionmesh_b200.preprocess import B200FramePreprocessor
    from actionmesh_b200.stage0 import TripoSGStage0

    root = st.write_tree(str(tmp_path_factory.mktemp("pretrained_weights")))
    stage0 = TripoSGStage0.from_pretrained(os.path.join(root, "TripoSG"), num_tokens=st.N_TOKENS)
    stage0.mesh_extractor = lambda lat: None
    image = B200FramePreprocessor().process_images(st.rgba_frames())[0]
    lats = [stage0(image, generator=torch.Generator(device="cuda").manual_seed(s), num_inference_steps=2,
                   guidance_scale=7.5)[0] for s in (44, 45)]
    st.centre_vae_field(root, lats)
    return root


def _frames_dir(tmp_path, n):
    d = tmp_path / f"frames_{n}"
    d.mkdir()
    for i, im in enumerate(st.rgba_frames(n)):
        im.save(d / f"{i}.png")
    return d


def _video_frames(path):
    import cv2

    cap, n, shape = cv2.VideoCapture(str(path)), 0, None
    while True:
        ok, fr = cap.read()
        if not ok:
            break
        n, shape = n + 1, fr.shape
    cap.release()
    return n, shape


FIRST_WINDOW = 16    # frames 0-15: the first AR window, decoded from the anchor mesh's own normals


def _check_outputs(out, meshes, want, faces):
    """The files in `out` hold `meshes`, what run_actionmesh returned, bit for bit; `meshes` equal `want`, the pipeline
    called directly.  Past the first AR window that holds to float rounding only: Stage II there reads the deformed anchor's
    vertex normals, summed with float atomics on the GPU in no fixed order (observed: up to 3.5e-6 on an H100, on meshes
    of extent ~0.5)."""
    from actionmesh_b200.gltf import load_glb, save_deformation

    assert len(meshes) == len(want)
    for i, (m, w) in enumerate(zip(meshes, want)):
        assert np.array_equal(m.faces, w.faces)
        if i < FIRST_WINDOW:
            assert np.array_equal(m.vertices, w.vertices), i
        else:
            err = np.abs(np.asarray(m.vertices, np.float64) - w.vertices).max()
            print(f"frame {i}: max |run_actionmesh - direct call| = {err:.3e}")
            assert err <= 1e-3 * np.abs(w.vertices).max(), (i, err)
        glb_check.check_glb(out / f"mesh_{i:02d}.glb")
        back = load_glb(out / f"mesh_{i:02d}.glb")
        assert np.array_equal(back.vertices, np.asarray(m.vertices).astype(np.float32)) and np.array_equal(back.faces, m.faces)
    vp, fp = save_deformation(meshes, out / "direct" / "deformations")
    for name, path in (("deformations_vertices.npy", vp), ("deformations_faces.npy", fp)):
        got, ref = np.load(out / name), np.load(path)
        assert got.dtype == ref.dtype and np.array_equal(got, ref)
    a = glb_check.check_animated(out / "animated_mesh.glb", np.stack([m.vertices for m in meshes]), faces)
    n, shape = _video_frames(out / "grid_normal.mp4")
    assert n == len(want) and shape == (256, 1024, 3)
    return a


@pytest.mark.parametrize("n_frames", [16, 20, 33])
def test_video_to_files(root, tmp_path, n_frames):
    """16 frames: one AR window; 20: two; 33: capped to 31 frames, as the reference's scripts load them."""
    from actionmesh_b200.inference import run_actionmesh
    from actionmesh_b200.pipeline import ActionMeshB200Pipeline
    from actionmesh_b200.video_input import load_frames

    frames = _frames_dir(tmp_path, n_frames)
    pipe = ActionMeshB200Pipeline.from_pretrained(root, config_updates=UPDATES).to("cuda")
    out = tmp_path / "out"
    meshes = run_actionmesh(pipe, str(frames), str(out), seed=44)
    want = pipe(load_frames(frames, max_frames=31), seed=44)
    assert len(want) == min(n_frames, 31) and len(want[0].faces) > 0
    _check_outputs(out, meshes, want, want[0].faces)


def _textured_sphere():
    from PIL import Image

    from actionmesh_b200.gltf import GltfVisual
    from actionmesh_b200.pipeline import Mesh

    n_lat, n_lon = 10, 14           # the closed UV sphere of test_mesh_input_pipeline_equals_injected
    th, ph = np.linspace(0, np.pi, n_lat + 1)[1:-1], np.linspace(0, 2 * np.pi, n_lon, endpoint=False)
    ring = np.stack([np.sin(th)[:, None] * np.cos(ph), np.sin(th)[:, None] * np.sin(ph),
                     np.cos(th)[:, None] * np.ones_like(ph)], -1).reshape(-1, 3) * 0.7
    v = np.concatenate([ring, [[0, 0, 0.7], [0, 0, -0.7]]])
    idx = lambda i, j: i * n_lon + j % n_lon
    f = [(idx(i, j), idx(i + 1, j), idx(i + 1, j + 1)) for i in range(n_lat - 2) for j in range(n_lon)]
    f += [(idx(i, j), idx(i + 1, j + 1), idx(i, j + 1)) for i in range(n_lat - 2) for j in range(n_lon)]
    top, bot = len(v) - 2, len(v) - 1
    f += [(top, idx(0, j), idx(0, j + 1)) for j in range(n_lon)] + [(bot, idx(n_lat - 2, j + 1), idx(n_lat - 2, j))
                                                                       for j in range(n_lon)]
    uv = np.stack([np.arctan2(v[:, 1], v[:, 0]) / (2 * np.pi) + 0.5, np.arccos(v[:, 2] / 0.7) / np.pi], -1)
    buf = io.BytesIO()
    Image.fromarray(np.random.default_rng(1).integers(0, 255, (16, 16, 3), dtype=np.uint8)).save(buf, format="PNG")
    visual = GltfVisual(uv=uv.astype(np.float32), material={"pbrMetallicRoughness": {"baseColorTexture": {"index": 0}}},
                        textures=[{"sampler": 0, "source": 0}], samplers=[{"magFilter": 9729}],
                        images=[{"mimeType": "image/png"}], image_bytes=[buf.getvalue()])
    return Mesh(vertices=v, faces=np.array(f, dtype=np.int64), visual=visual)


def test_mesh_input_to_files(root, tmp_path):
    from actionmesh_b200.gltf import load_glb, write_glb
    from actionmesh_b200.inference import run_actionmesh
    from actionmesh_b200.pipeline import ActionMeshB200PipelineWithMeshInput
    from actionmesh_b200.video_input import load_frames

    sphere = _textured_sphere()
    glb = tmp_path / "sphere.glb"
    write_glb(glb, sphere)
    frames = _frames_dir(tmp_path, 16)
    updates = {**UPDATES, "model.temporal_3D_denoiser.num_tokens_nominal": 2048}     # the VAE encoder's token count
    pipe = ActionMeshB200PipelineWithMeshInput.from_pretrained(root, config_updates=updates).to("cuda")
    out = tmp_path / "out"
    meshes = run_actionmesh(pipe, str(frames), str(out), seed=44, mesh_input=str(glb))
    want = pipe(load_frames(frames, max_frames=31), load_glb(glb), seed=44)
    assert all(np.array_equal(m.faces, sphere.faces) for m in meshes)
    a = _check_outputs(out, meshes, want, sphere.faces)
    assert np.array_equal(a["uv"], sphere.visual.uv) and a["image_bytes"] == sphere.visual.image_bytes
    assert a["material"] == sphere.visual.material
