"""Building the pipeline from the reference's checkpoint layout, without a GPU: the HF DinoV2 config mapping, the Stage 0
scheduler shift, and `from_pretrained`'s check that every required file exists before anything is loaded."""
import json
import os

import pytest

from actionmesh_b200 import AmbError

# (subdirectory, file) of every file ActionMeshB200Pipeline.from_pretrained needs, under the weights root
FILES = [("TripoSG/transformer", "config.json"), ("TripoSG/transformer", "diffusion_pytorch_model.safetensors"),
         ("TripoSG/vae", "config.json"), ("TripoSG/vae", "diffusion_pytorch_model.safetensors"),
         ("TripoSG/image_encoder_dinov2", "config.json"), ("TripoSG/image_encoder_dinov2", "model.safetensors"),
         ("TripoSG/feature_extractor_dinov2", "preprocessor_config.json"),
         ("TripoSG/scheduler", "scheduler_config.json"),
         ("dinov2", "config.json"), ("dinov2", "model.safetensors"), ("dinov2", "preprocessor_config.json"),
         ("RMBG", "model.safetensors"),
         ("ActionMesh/denoiser", "config.json"), ("ActionMesh/denoiser", "model.safetensors"),
         ("ActionMesh/autoencoder", "config.json"), ("ActionMesh/autoencoder", "model.safetensors")]


def _placeholder_tree(root, skip=None) -> str:
    """Every required file as an empty placeholder (only existence is checked before loading), except `skip`."""
    for d, f in FILES:
        if d == skip:
            continue
        os.makedirs(os.path.join(root, d), exist_ok=True)
        if (d, f) != skip:
            open(os.path.join(root, d, f), "w").close()
    return str(root)


def _dinov2(path, crop, shortest_edge=256):
    os.makedirs(path, exist_ok=True)
    cfg = {"model_type": "dinov2", "hidden_size": 512, "num_hidden_layers": 3, "num_attention_heads": 8, "image_size": 518,
           "patch_size": 14, "mlp_ratio": 4, "layer_norm_eps": 1e-6, "hidden_act": "gelu", "use_swiglu_ffn": False}
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump(cfg, f)
    pre = {"image_processor_type": "BitImageProcessor", "do_resize": True, "size": {"shortest_edge": shortest_edge},
           "resample": 3, "do_center_crop": True, "crop_size": {"height": crop, "width": crop}, "do_rescale": True,
           "rescale_factor": 1 / 255, "do_normalize": True, "image_mean": [0.485, 0.456, 0.406],
           "image_std": [0.229, 0.224, 0.225], "do_convert_rgb": True}
    with open(os.path.join(path, "preprocessor_config.json"), "w") as f:
        json.dump(pre, f)
    return str(path)


@pytest.mark.parametrize("crop", [224, 518])
def test_hf_dinov2_config_maps_layers_heads_and_crop(tmp_path, crop):
    from actionmesh_b200.image_encoder import hf_dinov2_arguments

    d = _dinov2(tmp_path / "dino", crop, shortest_edge=max(256, crop))
    args = hf_dinov2_arguments(d, d)
    assert args["num_layers"] == 3 and args["num_heads"] == 8 and args["hidden_size"] == 512
    assert args["image_size"] == crop          # the feature extractor's crop, not config.json's image_size (518)
    assert args["patch_size"] == 14 and args["mlp_ratio"] == 4 and args["layer_norm_eps"] == 1e-6


def test_hf_dinov2_config_rejects_crop_not_multiple_of_patch(tmp_path):
    from actionmesh_b200.image_encoder import hf_dinov2_arguments

    d = _dinov2(tmp_path / "dino", 200)
    with pytest.raises(AmbError, match="multiple of patch_size 14"):
        hf_dinov2_arguments(d, d)


def test_hf_dinov2_config_needs_both_files(tmp_path):
    from actionmesh_b200.image_encoder import hf_dinov2_arguments

    d = _dinov2(tmp_path / "dino", 224)
    os.remove(os.path.join(d, "preprocessor_config.json"))
    with pytest.raises(AmbError, match="preprocessor_config.json"):
        hf_dinov2_arguments(d, d)


def test_scheduler_shift_is_read_from_scheduler_config(tmp_path):
    from actionmesh_b200.stage0 import scheduler_shift

    with open(tmp_path / "scheduler_config.json", "w") as f:
        json.dump({"_class_name": "RectifiedFlowScheduler", "num_train_timesteps": 1000, "shift": 2.75}, f)
    assert scheduler_shift(str(tmp_path)) == 2.75
    with open(tmp_path / "scheduler_config.json", "w") as f:
        json.dump({"shift": 3.0, "use_dynamic_shifting": True}, f)
    with pytest.raises(AmbError, match="dynamic shifting"):
        scheduler_shift(str(tmp_path))
    os.remove(tmp_path / "scheduler_config.json")
    with pytest.raises(AmbError, match="scheduler_config.json"):
        scheduler_shift(str(tmp_path))


def test_from_pretrained_builds_the_reference_components_without_a_gpu(tmp_path):
    from actionmesh_b200.mesh_process import B200MeshPostprocessor
    from actionmesh_b200.pipeline import ActionMeshB200Pipeline, PassThroughMeshProcess
    from actionmesh_b200.preprocess import B200FramePreprocessor

    root = _placeholder_tree(tmp_path)
    pipe = ActionMeshB200Pipeline.from_pretrained(root, "actionmesh_b200_fast.yaml", lazy_loading=True)
    assert isinstance(pipe.mesh_process, B200MeshPostprocessor) and isinstance(pipe.image_process, B200FramePreprocessor)
    assert pipe.mesh_process.face_decimation == 40000 and pipe.mesh_process.floaters_threshold == 0.02
    assert pipe.cfg.stage_0_steps == 50 and pipe._actionmesh_weights_dir == os.path.join(root, "ActionMesh")
    assert sorted(pipe._loaders) == ["background_removal", "image_encoder", "image_to_3d_pipe"]
    # nothing is loaded until .to() or the stage that needs it
    assert all(getattr(pipe, a) is None for a in ("image_to_3d_pipe", "background_removal", "image_encoder",
                                                  "temporal_3D_denoiser", "temporal_3D_vae"))
    # the constructor is unchanged: pass-through post-processing, no loaders
    plain = ActionMeshB200Pipeline()
    assert isinstance(plain.mesh_process, PassThroughMeshProcess) and plain._loaders == {} and plain.image_process is None


@pytest.mark.parametrize("missing", sorted({d for d, _ in FILES} | {"TripoSG", "dinov2", "RMBG", "ActionMesh"}) + FILES)
def test_from_pretrained_names_the_missing_piece(tmp_path, missing):
    from actionmesh_b200.pipeline import ActionMeshB200Pipeline

    root = _placeholder_tree(tmp_path, skip=missing)
    if isinstance(missing, str) and "/" not in missing:            # a whole root directory
        import shutil

        shutil.rmtree(os.path.join(root, missing), ignore_errors=True)
    with pytest.raises(AmbError) as exc:
        ActionMeshB200Pipeline.from_pretrained(root)
    named = os.path.join(root, *(missing if isinstance(missing, tuple) else (missing,)))
    assert named in str(exc.value), (str(exc.value), named)


def test_mesh_input_pipeline_needs_only_triposg_vae(tmp_path):
    from actionmesh_b200.pipeline import ActionMeshB200PipelineWithMeshInput

    root = _placeholder_tree(tmp_path)
    for sub in ("transformer", "image_encoder_dinov2", "feature_extractor_dinov2", "scheduler"):
        import shutil

        shutil.rmtree(os.path.join(root, "TripoSG", sub))
    pipe = ActionMeshB200PipelineWithMeshInput.from_pretrained(root)
    assert "image_to_3d_pipe" not in pipe._loaders and pipe._triposg_weights_dir == os.path.join(root, "TripoSG")
    os.remove(os.path.join(root, "TripoSG", "vae", "diffusion_pytorch_model.safetensors"))
    with pytest.raises(AmbError, match="TripoSG/vae/diffusion_pytorch_model.safetensors"):
        ActionMeshB200PipelineWithMeshInput.from_pretrained(root)


def test_stage0_from_pretrained_checks_files_first(tmp_path):
    from actionmesh_b200.stage0 import TripoSGStage0

    root = _placeholder_tree(tmp_path, skip=("TripoSG/scheduler", "scheduler_config.json"))
    with pytest.raises(AmbError, match="TripoSG/scheduler/scheduler_config.json"):
        TripoSGStage0.from_pretrained(os.path.join(root, "TripoSG"))
