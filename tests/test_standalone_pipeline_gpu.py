"""The pipeline built from a checkpoint directory (-m gpu): `TripoSGStage0.from_pretrained` and
`ActionMeshB200Pipeline(WithMeshInput).from_pretrained` on a tiny tree in the reference's layout (tests/standalone_tree.py)
give bit for bit what the same files give when the components are built by hand and injected."""
import os

import numpy as np
import pytest
import torch

import standalone_tree as st

pytestmark = pytest.mark.gpu

STEPS0 = 2
UPDATES = {"model.temporal_3D_denoiser.num_tokens_nominal": st.N_TOKENS, "stage_0_steps": STEPS0, "stage_1_steps": 2}
POSTPROCESS = {"model.mesh_process._target_": "actionmesh_b200.mesh_process.B200MeshPostprocessor"}


def _crop_anchor(frames):
    from actionmesh_b200.preprocess import B200FramePreprocessor

    return B200FramePreprocessor().process_images(frames)[0]


@pytest.fixture(scope="module")
def trees(tmp_path_factory, amb_lib):
    """{224: full tree, 518: a TripoSG directory whose DinoV2 crops 518}; the VAE's field is centred on the anchor latents
    of seeds 44 and 45 so that Stage 0 yields a surface."""
    from actionmesh_b200.stage0 import TripoSGStage0

    root = st.write_tree(str(tmp_path_factory.mktemp("pretrained_weights")))
    stage0 = TripoSGStage0.from_pretrained(os.path.join(root, "TripoSG"), num_tokens=st.N_TOKENS)
    stage0.mesh_extractor = lambda lat: None
    image = _crop_anchor(st.rgba_frames())
    lats = [stage0(image, generator=torch.Generator(device="cuda").manual_seed(s), num_inference_steps=STEPS0,
                   guidance_scale=7.5)[0] for s in (44, 45)]
    sd = st.centre_vae_field(root, lats)
    tri518 = os.path.join(str(tmp_path_factory.mktemp("triposg518")), "TripoSG")
    st.write_triposg(tri518, crop=518)
    st.write_vae(tri518, sd)
    return {224: root, 518: os.path.dirname(tri518)}


def _manual_stage0(triposg_dir, crop):
    """TripoSGStage0 assembled by hand from the files, with the shapes written out."""
    from safetensors.torch import load_file

    from actionmesh_b200.image_encoder import B200ImageEncoder
    from actionmesh_b200.stage0 import B200TripoSGDiT, TripoSGStage0
    from actionmesh_b200.triposg_vae import B200TripoSGVAE

    dit = B200TripoSGDiT(**st.DIT).to("cuda")
    dit.load_state_dict(load_file(os.path.join(triposg_dir, "transformer", "diffusion_pytorch_model.safetensors")))
    vae = B200TripoSGVAE(**st.VAE).to("cuda")
    vae.load_state_dict(load_file(os.path.join(triposg_dir, "vae", "diffusion_pytorch_model.safetensors")))
    enc = B200ImageEncoder(os.path.join(triposg_dir, "feature_extractor_dinov2"), os.path.join(triposg_dir, "image_encoder_dinov2"),
                           **st.DINO, image_size=crop, precision="bf16").to("cuda")
    return TripoSGStage0(dit, enc, mesh_extractor=vae.extract_mesh, shift=st.SHIFT, num_tokens=st.N_TOKENS)


def _injected(root, cls=None, **updates):
    """The pipeline constructed the existing way, the same components injected."""
    from actionmesh_b200.background_removal import B200BackgroundRemover
    from actionmesh_b200.image_encoder import B200ImageEncoder
    from actionmesh_b200.pipeline import ActionMeshB200Pipeline
    from actionmesh_b200.preprocess import B200FramePreprocessor

    cls = cls or ActionMeshB200Pipeline
    kw = dict(background_removal=B200BackgroundRemover(os.path.join(root, "RMBG")), image_process=B200FramePreprocessor(),
              weights_dir=os.path.join(root, "ActionMesh"), config_updates={**UPDATES, **POSTPROCESS, **updates})
    if cls is ActionMeshB200Pipeline:
        kw["image_to_3d"] = _manual_stage0(os.path.join(root, "TripoSG"), 224)
    else:
        kw["triposg_weights_dir"] = os.path.join(root, "TripoSG")
    pipe = cls("actionmesh_b200.yaml", **kw)
    dino = os.path.join(root, "dinov2")
    pipe.image_encoder = B200ImageEncoder(dino, dino, **st.DINO).to("cuda")
    return pipe.to("cuda")


def _input(frames):
    from actionmesh_b200.pipeline import ActionMeshInput

    return ActionMeshInput(list(frames), torch.arange(len(frames), dtype=torch.float32))


def _same(a, b) -> bool:
    return len(a) == len(b) and all(np.array_equal(np.asarray(x.vertices), np.asarray(y.vertices))
                                    and np.array_equal(np.asarray(x.faces), np.asarray(y.faces)) for x, y in zip(a, b))


@pytest.mark.parametrize("crop", [224, 518])
def test_stage0_loader_equals_manual_assembly(trees, crop):
    from actionmesh_b200.stage0 import TripoSGStage0

    triposg_dir = os.path.join(trees[crop], "TripoSG")
    image = _crop_anchor(st.rgba_frames())
    auto = TripoSGStage0.from_pretrained(triposg_dir, num_tokens=st.N_TOKENS)
    assert auto.shift == st.SHIFT and auto.image_encoder.precision == "bf16" and auto.image_encoder.image_size == crop
    run = lambda s0: s0(image, generator=torch.Generator(device="cuda").manual_seed(44), num_inference_steps=STEPS0,
                        guidance_scale=7.5)
    lat, mesh = run(auto)
    ref_lat, ref_mesh = run(_manual_stage0(triposg_dir, crop))
    assert torch.equal(lat, ref_lat)
    assert np.array_equal(mesh.vertices, ref_mesh.vertices) and np.array_equal(mesh.faces, ref_mesh.faces)
    if crop == 224:
        assert len(mesh.faces) > 0
    else:
        assert auto.image_encoder.encode_images([image]).shape == (1, 1 + (crop // 14) ** 2, st.DINO["hidden_size"])


@pytest.mark.parametrize("lazy", [False, True])
def test_standalone_pipeline_equals_injected_pipeline(trees, lazy):
    from actionmesh_b200.pipeline import ActionMeshB200Pipeline

    root = trees[224]
    frames = st.rgba_frames()
    pipe = ActionMeshB200Pipeline.from_pretrained(root, lazy_loading=lazy, config_updates=UPDATES).to("cuda")
    meshes = pipe(_input(frames), seed=44)
    assert len(meshes) == len(frames) and len(meshes[0].faces) > 0
    assert _same(meshes, _injected(root)(_input(frames), seed=44))
    if lazy:
        assert all(getattr(pipe, a) is None for a in ("background_removal", "image_to_3d_pipe", "image_encoder",
                                                      "temporal_3D_denoiser", "temporal_3D_vae"))


def test_mesh_postprocessing_runs(trees):
    from actionmesh_b200.mesh_process import B200MeshPostprocessor
    from actionmesh_b200.pipeline import ActionMeshB200Pipeline

    root = trees[224]
    frames = st.rgba_frames()
    _, anchor = _manual_stage0(os.path.join(root, "TripoSG"), 224)(
        _crop_anchor(frames), generator=torch.Generator(device="cuda").manual_seed(44), num_inference_steps=STEPS0,
        guidance_scale=7.5)
    target = len(anchor.faces) // 2          # well below the default 40 000, and reachable on this surface
    meshes = ActionMeshB200Pipeline.from_pretrained(root, config_updates=UPDATES).to("cuda")(_input(frames), seed=44,
                                                                                             face_decimation=target)
    post = B200MeshPostprocessor(face_decimation=target, floaters_threshold=0.02).process_mesh(anchor)
    assert all(np.array_equal(m.faces, post.faces) for m in meshes)
    assert 0 < len(meshes[0].faces) <= target


def test_background_removal_is_wired(trees):
    from PIL import Image

    import rmbg_ref
    from actionmesh_b200.background_removal import B200BackgroundRemover
    from actionmesh_b200.pipeline import ActionMeshB200Pipeline

    root = trees[224]
    frames = [Image.fromarray(rmbg_ref.synthetic_frame(120, 160, seed=i), "RGB") for i in range(16)]
    pipe = ActionMeshB200Pipeline.from_pretrained(root, config_updates=UPDATES).to("cuda")
    seen = []

    class Stop(Exception):
        pass

    def capture(images):          # what reaches the cropping step is what the pipeline's remover returned
        seen.extend(images)
        raise Stop

    pipe.image_process.process_images = capture
    with pytest.raises(Stop):
        pipe(_input(frames), seed=44)
    want = B200BackgroundRemover(os.path.join(root, "RMBG")).process_images(frames)
    assert len(seen) == len(want) and all(im.mode == "RGBA" for im in seen)
    assert all(np.array_equal(np.asarray(a), np.asarray(b)) for a, b in zip(seen, want))


def test_seeds(trees):
    from actionmesh_b200.pipeline import ActionMeshB200Pipeline

    frames = st.rgba_frames()
    pipe = ActionMeshB200Pipeline.from_pretrained(trees[224], config_updates=UPDATES).to("cuda")
    a, b, c = (pipe(_input(frames), seed=s) for s in (44, 44, 45))
    assert _same(a, b)
    assert not _same(a, c)


def test_mesh_input_pipeline_equals_injected(trees):
    from actionmesh_b200.pipeline import ActionMeshB200PipelineWithMeshInput, Mesh

    root = trees[224]
    n_lat, n_lon = 10, 14           # a closed UV sphere
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
    f = np.array(f, dtype=np.int64)
    updates = {"model.temporal_3D_denoiser.num_tokens_nominal": 2048}     # the VAE encoder's token count
    frames = st.rgba_frames()
    run = lambda p: p(_input(frames), Mesh(vertices=v.copy(), faces=f.copy()), seed=44)
    pipe = ActionMeshB200PipelineWithMeshInput.from_pretrained(root, config_updates={**UPDATES, **updates}).to("cuda")
    meshes = run(pipe)
    assert len(meshes) == len(frames) and np.array_equal(meshes[0].faces, f)
    assert _same(meshes, run(_injected(root, ActionMeshB200PipelineWithMeshInput, **updates)))
