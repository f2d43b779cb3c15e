"""The command line: video (+ optional .glb mesh) -> animated meshes on disk, on this package alone.

    python -m actionmesh_b200.inference --input clip.mp4 [--mesh_input mesh.glb] [--output_dir DIR] [--fast] [--low_ram]
                                        [--render_texture] [--skinning_bones N] [--keep_rig] [--auto_rig N]

One entry point for the reference's `inference/video_to_animated_mesh.py` and `inference/video_and_3d_to_animated_mesh.py`
(`--mesh_input` selects the second), with their flags and defaults plus `--weights_root`.  It writes, in `--output_dir`
(default outputs/<input stem>): mesh_00.glb ..., deformations_vertices.npy, deformations_faces.npy, animated_mesh.glb and
grid_normal.mp4, and with `--render_texture` also grid_texture.mp4 (the meshes shaded with the input mesh's texture, or
with the default colour), and with `--skinning_bones N` also skinned_mesh.glb (the same animation as N bones and skin
weights fitted on the GPU, `skinning.fit_skinning`), and with `--keep_rig` (a rigged `--mesh_input`) also rigged_mesh.glb (the
input file with its own skeleton animated: joint rotations fitted on the GPU, `rig.fit_rig_animation`), and with
`--auto_rig N` also auto_rigged_mesh.glb (a skeleton of N joints found from the animation itself, its joint rotations
and skin weights fitted on the GPU, `autorig.fit_auto_rig`).  `--blender_path` and `--dtype` are accepted so that the reference's documented command lines run
unchanged, and have no effect: the animated GLB is written without Blender, and the CUDA path owns its precision.
"""
from __future__ import annotations

import argparse
import copy
import logging
import os
from pathlib import Path
from typing import Optional

import numpy as np
import torch

from . import autorig, render
from . import rig as rig_fit
from . import skinning
from .gltf import GltfRig, load_glb, load_rig, save_deformation, save_meshes, write_animated_glb, write_rig_animation, \
    write_auto_rig_glb, write_skinned_glb
from .pipeline import ActionMeshB200Pipeline, ActionMeshB200PipelineWithMeshInput
from .video_input import load_frames

logger = logging.getLogger(__name__)

MAX_FRAMES = 31      # both reference scripts load at most 31 frames
ANIMATION_FPS = 8


@torch.no_grad()
def run_actionmesh(pipeline, input: str, output_dir: str, seed: int = 44, mesh_input: Optional[str] = None,
                   render_texture: bool = False, skinning_bones: int = 0, rig: Optional[GltfRig] = None,
                   auto_rig_joints: int = 0, **overrides) -> list:
    """The reference scripts' `run_actionmesh`: load the frames (and the mesh), run `pipeline`, write every output file
    into `output_dir` -> the meshes.  `render_texture` adds grid_texture.mp4, shaded with the input mesh's visual (the one
    the animated GLB gets).  `skinning_bones` > 0 adds skinned_mesh.glb: that many bones fitted to the animated GLB's
    vertices, written with its faces and visual.  `rig` (`load_rig(mesh_input)`) adds rigged_mesh.glb: the input file with
    its joint rotations fitted to the same vertices.  `auto_rig_joints` > 0 adds auto_rigged_mesh.glb: a skeleton of that
    many joints found from the same vertices and faces, written with the visual.  `overrides` are the pipeline's per-call arguments (stage_0_steps, face_decimation,
    floaters_threshold, stage_1_steps, guidance_scales, anchor_idx)."""
    frames = load_frames(input, max_frames=MAX_FRAMES)
    visual = None
    if mesh_input is None:
        meshes = pipeline(input=frames, seed=seed, **overrides)
        faces = np.asarray(meshes[0].faces)
    else:
        anchor_mesh = load_glb(mesh_input)
        # the pipeline merges the mesh's vertices in place: keep what the animated GLB needs first
        visual = copy.deepcopy(anchor_mesh.visual)
        faces = np.array(anchor_mesh.faces, copy=True)
        meshes = pipeline(input=frames, anchor_mesh=anchor_mesh, seed=seed, **overrides)
    os.makedirs(output_dir, exist_ok=True)
    save_meshes(meshes, output_dir)
    save_deformation(meshes, os.path.join(output_dir, "deformations"))
    animated = os.path.join(output_dir, "animated_mesh.glb")
    vertices = np.stack([np.asarray(m.vertices) for m in meshes])
    write_animated_glb(animated, vertices, faces, fps=ANIMATION_FPS, visual=visual)
    logger.info(f"Animated GLB saved to {animated}")
    if skinning_bones > 0:
        fit = skinning.fit_skinning(vertices, skinning_bones, device=pipeline.device)
        skinned = os.path.join(output_dir, "skinned_mesh.glb")
        write_skinned_glb(skinned, fit, faces, fps=ANIMATION_FPS, visual=visual)
        logger.info(f"Skinned GLB saved to {skinned} ({skinning_bones} bones; RMS error {fit.rms_error:.3e}, max error "
                    f"{fit.max_error:.3e} of the rest bounding-box diagonal)")
    if rig is not None:
        if mesh_input is None:
            raise ValueError("a rig is kept only for a --mesh_input")
        fit = rig_fit.fit_rig_animation(rig, vertices, device=pipeline.device)
        rigged = os.path.join(output_dir, "rigged_mesh.glb")
        write_rig_animation(mesh_input, rigged, rig, fit, fps=ANIMATION_FPS)
        logger.info(f"Rigged GLB saved to {rigged} ({len(rig.joint_nodes)} joints; RMS error {fit.rms_error:.3e}, max error "
                    f"{fit.max_error:.3e} of the rest bounding-box diagonal)")
    if auto_rig_joints > 0:
        fit = autorig.fit_auto_rig(vertices, faces, auto_rig_joints, device=pipeline.device)
        auto_rigged = os.path.join(output_dir, "auto_rigged_mesh.glb")
        write_auto_rig_glb(auto_rigged, fit, faces, fps=ANIMATION_FPS, visual=visual)
        logger.info(f"Auto-rigged GLB saved to {auto_rigged} ({auto_rig_joints} joints; RMS error {fit.rms_error:.3e} against "
                    f"{fit.ssdr_rms_error:.3e} for flat bones, max error {fit.max_error:.3e} of the rest bounding-box "
                    f"diagonal)")
    visualizer = render.B200MeshVisualizer(image_size=256)
    if render_texture:
        visualizer.render(meshes, pipeline.device, output_dir, frames.frames, modalities=("normal", "texture"),
                          visual=visual)
    else:
        visualizer.render(meshes, pipeline.device, output_dir, frames.frames)
    return meshes


def parse_args(argv=None) -> argparse.Namespace:
    p = argparse.ArgumentParser(prog="python -m actionmesh_b200.inference", description=__doc__.split("\n\n")[0])
    p.add_argument("--input", type=str, required=True, help="Input video (.mp4, .avi, .mov), image glob or directory.")
    p.add_argument("--mesh_input", type=str, default=None,
                   help="Anchor mesh (.glb): animate this mesh instead of generating one from the anchor frame.")
    p.add_argument("--output_dir", type=str, default=None, help="Default: outputs/<input stem>.")
    p.add_argument("--seed", type=int, default=44)
    p.add_argument("--weights_root", type=str, default="pretrained_weights",
                   help="Directory holding TripoSG/, dinov2/, RMBG/ and ActionMesh/.")
    p.add_argument("--blender_path", type=str, default=None, help="Accepted for compatibility; not needed.")
    p.add_argument("--fast", action="store_true", help="Fast preset (stage_0_steps=50, stage_1_steps=15).")
    p.add_argument("--low_ram", action="store_true", help="Load each model just before its stage, release it after.")
    p.add_argument("--dtype", type=str, choices=["bfloat16", "float16"], default="bfloat16",
                   help="Accepted for compatibility; the CUDA path owns its precision.")
    p.add_argument("--stage_0_steps", type=int, default=None, help="Image-to-3D (TripoSG) steps. Default: 100. Fast: 50")
    p.add_argument("--face_decimation", type=int, default=None, help="Target faces of the anchor mesh. Default: 40000")
    p.add_argument("--floaters_threshold", type=float, default=None, help="Floater removal threshold. Default: 0.02")
    p.add_argument("--stage_1_steps", type=int, default=None, help="Stage I denoising steps. Default: 30. Fast: 15")
    p.add_argument("--guidance_scales", type=float, nargs="+", default=None, help="Stage I CFG scales. Default: [7.5]")
    p.add_argument("--anchor_idx", type=int, default=None, help="Index of the anchor frame. Default: 0")
    p.add_argument("--render_texture", action="store_true",
                   help="Also write grid_texture.mp4: the meshes shaded with the input mesh's texture (or a flat colour).")
    p.add_argument("--skinning_bones", type=int, default=0,
                   help="Also write skinned_mesh.glb with this many bones fitted to the animation (at most 256). Default: 0 (off)")
    p.add_argument("--keep_rig", action="store_true",
                   help="Also write rigged_mesh.glb: the rigged --mesh_input with its own skeleton animated.")
    p.add_argument("--auto_rig", type=int, default=0, metavar="N",
                   help="Also write auto_rigged_mesh.glb: a skeleton of N joints found from the animation, its joint "
                        "rotations and skin weights fitted to it (at most 256). Default: 0 (off)")
    args = p.parse_args(argv)
    if not 0 <= args.auto_rig <= 256:
        p.error(f"--auto_rig must be in [0, 256], got {args.auto_rig}")
    if args.keep_rig and args.mesh_input is None:
        p.error("--keep_rig needs --mesh_input (a rigged .glb)")
    return args


def main(argv=None) -> list:
    logging.basicConfig(level=logging.INFO, format="%(asctime)s - %(name)s - %(levelname)s - %(message)s")
    args = parse_args(argv)
    if args.blender_path is not None:
        logger.info("--blender_path has no effect: animated_mesh.glb is written without Blender")
    if args.dtype != "bfloat16":
        logger.info(f"--dtype {args.dtype} has no effect: the CUDA path owns its precision")
    rig = None
    if args.keep_rig:
        try:
            rig = load_rig(args.mesh_input)        # before any model loads: a file without a usable rig fails fast
        except ValueError as exc:
            raise SystemExit(f"--keep_rig: {exc}") from exc
    config_name = "actionmesh_b200_fast.yaml" if args.fast else "actionmesh_b200.yaml"
    output_dir = args.output_dir or f"outputs/{Path(args.input).stem}"
    cls = ActionMeshB200Pipeline if args.mesh_input is None else ActionMeshB200PipelineWithMeshInput
    pipeline = cls.from_pretrained(args.weights_root, config_name=config_name, lazy_loading=args.low_ram).to("cuda")
    overrides = {k: getattr(args, k) for k in ("stage_0_steps", "face_decimation", "floaters_threshold",
                                               "stage_1_steps", "guidance_scales", "anchor_idx")}
    return run_actionmesh(pipeline, args.input, output_dir, seed=args.seed, mesh_input=args.mesh_input,
                          render_texture=args.render_texture, skinning_bones=args.skinning_bones, rig=rig,
                          auto_rig_joints=args.auto_rig, **overrides)


if __name__ == "__main__":
    main()
