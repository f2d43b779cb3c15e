"""The command line (`python -m actionmesh_b200.inference`) with the pipelines and the renderer stubbed: flags reach the
pipeline's construction and call, and the output directory holds the reference's files."""
import os

import numpy as np
import pytest
import torch
from PIL import Image

import glb_check
from actionmesh_b200 import inference, render
from actionmesh_b200.gltf import GltfVisual, load_glb, write_glb
from actionmesh_b200.pipeline import ActionMeshB200Pipeline, ActionMeshB200PipelineWithMeshInput, Mesh

N_VERTS, N_FACES = 40, 60


class StubPipeline:
    """Records how it was built and called; returns seeded meshes on one set of faces (the input mesh's, if any)."""

    def __init__(self, cls, args, kwargs):
        self.cls, self.args, self.kwargs, self.calls, self.device = cls, args, kwargs, [], None

    def to(self, device):
        self.device = torch.device(device)
        return self

    def __call__(self, input, seed=44, anchor_mesh=None, **overrides):
        self.calls.append(dict(input=input, seed=seed, anchor_mesh=anchor_mesh, **overrides))
        rng = np.random.default_rng(seed)
        if anchor_mesh is None:
            verts, faces = rng.standard_normal((N_VERTS, 3)), rng.integers(0, N_VERTS, (N_FACES, 3))
        else:
            verts, faces = np.asarray(anchor_mesh.vertices), np.array(anchor_mesh.faces)
            anchor_mesh.faces, anchor_mesh.visual = faces[:1], None        # the real pipeline edits the mesh in place
        return [Mesh(vertices=verts + 0.01 * k * rng.standard_normal(verts.shape), faces=faces)
                for k in range(input.n_frames)]


@pytest.fixture
def stubs(monkeypatch):
    built, rendered = [], []

    def factory(cls):
        def from_pretrained(*args, **kwargs):
            built.append(StubPipeline(cls, args, kwargs))
            return built[-1]
        return from_pretrained

    class Visualizer:
        def __init__(self, image_size=256):
            self.image_size = image_size

        def render(self, meshes, device, output_dir, input_frames):
            rendered.append(dict(image_size=self.image_size, meshes=meshes, device=device, output_dir=output_dir,
                                 input_frames=input_frames))

    for cls in (ActionMeshB200Pipeline, ActionMeshB200PipelineWithMeshInput):
        monkeypatch.setattr(cls, "from_pretrained", classmethod(lambda c, *a, **k: factory(c)(*a, **k)))
    monkeypatch.setattr(render, "B200MeshVisualizer", Visualizer)
    return built, rendered


@pytest.fixture
def frames_dir(tmp_path):
    d = tmp_path / "clip"
    d.mkdir()
    for i in range(18):
        Image.fromarray(np.random.default_rng(i).integers(0, 255, (32, 32, 4), dtype=np.uint8), "RGBA").save(d / f"{i}.png")
    return d


@pytest.mark.parametrize("flags,config_name,lazy", [([], "actionmesh_b200.yaml", False),
                                                    (["--fast"], "actionmesh_b200_fast.yaml", False),
                                                    (["--low_ram"], "actionmesh_b200.yaml", True),
                                                    (["--fast", "--low_ram"], "actionmesh_b200_fast.yaml", True)])
def test_flags_select_config_and_lazy_loading(stubs, frames_dir, tmp_path, flags, config_name, lazy):
    built, _ = stubs
    inference.main(["--input", str(frames_dir), "--output_dir", str(tmp_path / "out"), *flags])
    (pipe,) = built
    assert pipe.cls is ActionMeshB200Pipeline and pipe.device == torch.device("cuda")
    assert pipe.args == ("pretrained_weights",) and pipe.kwargs == {"config_name": config_name, "lazy_loading": lazy}


def test_overrides_reach_the_call(stubs, frames_dir, tmp_path):
    built, rendered = stubs
    inference.main(["--input", str(frames_dir), "--output_dir", str(tmp_path / "out"), "--seed", "7",
                    "--weights_root", "/w", "--stage_0_steps", "3", "--face_decimation", "500",
                    "--floaters_threshold", "0.1", "--stage_1_steps", "4", "--guidance_scales", "2.0", "3.5",
                    "--anchor_idx", "2", "--blender_path", "/opt/blender/blender", "--dtype", "float16"])
    (pipe,) = built
    assert pipe.args == ("/w",)
    (call,) = pipe.calls
    assert call["seed"] == 7 and call["anchor_mesh"] is None and call["input"].n_frames == 18
    assert {k: call[k] for k in ("stage_0_steps", "face_decimation", "floaters_threshold", "stage_1_steps",
                                 "guidance_scales", "anchor_idx")} == dict(
        stage_0_steps=3, face_decimation=500, floaters_threshold=0.1, stage_1_steps=4, guidance_scales=[2.0, 3.5],
        anchor_idx=2)
    (r,) = rendered
    assert r["image_size"] == 256 and r["device"] == torch.device("cuda") and r["output_dir"] == str(tmp_path / "out")
    assert r["input_frames"] is call["input"].frames and len(r["meshes"]) == 18


def test_defaults(stubs, frames_dir, tmp_path, monkeypatch):
    built, _ = stubs
    monkeypatch.chdir(tmp_path)
    inference.main(["--input", str(frames_dir)])
    (call,) = built[0].calls
    assert call["seed"] == 44 and all(call[k] is None for k in ("stage_0_steps", "face_decimation", "floaters_threshold",
                                                                 "stage_1_steps", "guidance_scales", "anchor_idx"))
    assert sorted(os.listdir(tmp_path / "outputs")) == ["clip"]


def test_output_files(stubs, frames_dir, tmp_path):
    built, _ = stubs
    out = tmp_path / "out"
    meshes = inference.main(["--input", str(frames_dir), "--output_dir", str(out)])
    assert sorted(os.listdir(out)) == sorted([f"mesh_{i:02d}.glb" for i in range(18)] + [
        "deformations_vertices.npy", "deformations_faces.npy", "animated_mesh.glb"])
    for i, m in enumerate(meshes):
        glb_check.check_glb(out / f"mesh_{i:02d}.glb")
        back = load_glb(out / f"mesh_{i:02d}.glb")
        assert np.array_equal(back.vertices, m.vertices.astype(np.float32)) and np.array_equal(back.faces, m.faces)
    v = np.load(out / "deformations_vertices.npy")
    assert v.shape == (18, N_VERTS, 3) and np.array_equal(np.load(out / "deformations_faces.npy"), meshes[0].faces)
    glb_check.check_animated(out / "animated_mesh.glb", np.stack([m.vertices for m in meshes]), meshes[0].faces)


def test_mesh_input(stubs, frames_dir, tmp_path):
    built, _ = stubs
    rng = np.random.default_rng(5)
    png = b"\x89PNG\r\n\x1a\n" + bytes(rng.integers(0, 255, 61, dtype=np.uint8))
    visual = GltfVisual(uv=rng.random((N_VERTS, 2)).astype(np.float32),
                        material={"pbrMetallicRoughness": {"baseColorTexture": {"index": 0}}},
                        textures=[{"source": 0}], images=[{"mimeType": "image/png"}], image_bytes=[png])
    faces = rng.integers(0, N_VERTS, (N_FACES, 3))
    write_glb(tmp_path / "in.glb", Mesh(vertices=rng.standard_normal((N_VERTS, 3)), faces=faces, visual=visual))
    out = tmp_path / "out"
    meshes = inference.main(["--input", str(frames_dir), "--mesh_input", str(tmp_path / "in.glb"),
                             "--output_dir", str(out)])
    (pipe,) = built
    assert pipe.cls is ActionMeshB200PipelineWithMeshInput
    assert np.array_equal(pipe.calls[0]["anchor_mesh"].faces, faces[:1])      # edited in place by the pipeline ...
    a = glb_check.check_animated(out / "animated_mesh.glb", np.stack([m.vertices for m in meshes]), faces)
    assert np.array_equal(a["uv"], visual.uv) and a["image_bytes"] == [png]    # ... but not in the animated GLB
    assert a["material"] == visual.material
