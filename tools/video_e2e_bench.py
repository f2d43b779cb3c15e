"""Seconds per video of the whole video -> 4D call, `ActionMeshB200Pipeline.__call__`, per stage, for actionmesh_b200.yaml and
actionmesh_b200_fast.yaml.  Prints one JSON line.

Inputs: the random-frame video of SURVEY section 8(d) (16 frames, 512 x 512 uniform RGB from seed 7, alpha = centred disc of
radius 180 px) and full-size models with seeded random weights, assigned directly (no checkpoints are read).  The frames have
a valid alpha, so background removal passes them through, as it does for the reference.

Random weights make the Stage 0 surface arbitrary, and post-processing and Stage II time depend on its size.  The TripoSG VAE
uses the weights of `tools/gpu_probe.py vae_decode` (triposg_vae_ref.make_state_dict(1024, 8, 16, seed=1)) with two changes,
so that a surface of a real object's scale comes out: proj_query keeps only its raw-coordinate columns (the frequency columns
would make the random field a foam of tens of millions of faces at octree depth 9), and proj_out's bias is shifted so that
the field of this video's anchor latent is zero at its median over a 64^3 grid.  The anchor mesh's vertex and face counts
before and after post-processing are reported with the times.

Each stage is timed with a host clock after a device synchronise.  One warm-up call, then three timed calls per config.

    python tools/video_e2e_bench.py [--calls 3] [--out /tmp/video_e2e.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

CONFIGS = ("actionmesh_b200.yaml", "actionmesh_b200_fast.yaml")
STAGES = ("background_removal", "crop", "stage0_dinov2", "stage0_dit", "stage0_vae_dmc", "postprocess", "dinov2",
          "stage1", "stage2")


def gpu_card() -> dict:
    """Name and power limit of the GPU, read with a query (no setting is changed)."""
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, check=True).stdout.strip().splitlines()[0]
    name, power = (s.strip() for s in out.split(","))
    return {"name": name, "power_limit": power}


def frames(n: int = 16, size: int = 512, radius: int = 180, seed: int = 7) -> list:
    import numpy as np
    from PIL import Image

    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:size, 0:size]
    alpha = np.where((x - size / 2) ** 2 + (y - size / 2) ** 2 < radius ** 2, 255, 0).astype(np.uint8)
    return [Image.fromarray(np.dstack([rng.integers(0, 256, (size, size, 3), dtype=np.uint8), alpha]), "RGBA")
            for _ in range(n)]


class Timer:
    """Host-clock time per stage, each taken after a device synchronise."""

    def __init__(self):
        self.t: dict = {}

    def wrap(self, name: str, fn):
        import torch

        def timed(*args, **kwargs):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = fn(*args, **kwargs)
            torch.cuda.synchronize()
            self.t[name] = self.t.get(name, 0.0) + time.perf_counter() - t0
            return out

        return timed


def build_models():
    import rmbg_ref
    import triposg_vae_ref as vref
    from actionmesh_b200.autoencoder import B200Autoencoder
    from actionmesh_b200.background_removal import B200BackgroundRemover
    from actionmesh_b200.denoiser import B200Denoiser, DenoiserConfig
    from actionmesh_b200.image_encoder import B200ImageEncoder
    from actionmesh_b200.stage0 import B200TripoSGDiT, TripoSGStage0
    from actionmesh_b200.triposg_vae import B200TripoSGVAE

    m = {}
    m["rmbg"] = B200BackgroundRemover().to("cuda")
    m["rmbg"].load_state_dict(rmbg_ref.make_state_dict(0, device="cuda"))
    dit = B200TripoSGDiT().to("cuda")
    dit.init_random_(seed=1238)
    tri_enc = B200ImageEncoder(precision="bf16").to("cuda")   # Stage 0's rule: bf16 operands (DESIGN section 18)
    tri_enc.init_random_(seed=1239)
    vae_sd = vref.make_state_dict(1024, 8, 16, seed=1)
    vae_sd["decoder.proj_query.weight"][:, 3:] = 0.0            # raw coordinates only: a smooth random field
    vae = B200TripoSGVAE().to("cuda")
    vae.load_state_dict(vae_sd)
    m["vae"], m["vae_sd"] = vae, vae_sd
    m["stage0"] = TripoSGStage0(dit, tri_enc, mesh_extractor=vae.extract_mesh, shift=1.0, num_tokens=2048)
    m["dinov2"] = B200ImageEncoder().to("cuda")
    m["dinov2"].init_random_(seed=1235)
    m["denoiser"] = B200Denoiser(DenoiserConfig()).to("cuda")
    m["denoiser"].init_random_(seed=1234)
    m["autoencoder"] = B200Autoencoder().to("cuda")
    m["autoencoder"].init_random_(seed=1236)
    return m


def centre_field(m: dict, image, steps: int) -> None:
    """Shift the VAE's proj_out bias to the median of the anchor latent's field over a 64^3 grid."""
    import torch

    lat = m["stage0"].denoise(m["stage0"].image_encoder.encode_images([image]),
                              torch.randn((1, 2048, 64), generator=torch.Generator(device="cuda").manual_seed(44),
                                          device="cuda"), steps, 7.5)
    a = torch.linspace(-1.005, 1.005, 64, device="cuda")
    xyz = torch.stack(torch.meshgrid(a, a, a, indexing="ij"), -1).reshape(-1, 3)
    vae = m["vae"]
    med = vae.query(vae.prepare(lat[0]), xyz)[:, 0].median().cpu()
    m["vae_sd"]["decoder.proj_out.bias"] = m["vae_sd"]["decoder.proj_out.bias"] + med
    vae.load_state_dict(m["vae_sd"])


def run_config(m: dict, config: str, calls: int) -> dict:
    import torch

    from actionmesh_b200.pipeline import ActionMeshB200Pipeline, ActionMeshInput, AnimationPipeline
    from actionmesh_b200.preprocess import B200FramePreprocessor

    pipe = ActionMeshB200Pipeline(config, image_to_3d=m["stage0"], background_removal=m["rmbg"],
                                  image_process=B200FramePreprocessor(),
                                  config_updates={"model.mesh_process._target_":
                                                  "actionmesh_b200.mesh_process.B200MeshPostprocessor"})
    pipe.image_encoder, pipe.temporal_3D_denoiser, pipe.temporal_3D_vae = m["dinov2"], m["denoiser"], m["autoencoder"]
    pipe.to("cuda")
    timer = Timer()
    s0 = m["stage0"]
    originals = {"rmbg": m["rmbg"].process_images, "crop": pipe.image_process.process_images,
                 "s0_enc": s0.image_encoder.encode_images, "s0_denoise": s0.denoise, "s0_mesh": s0.mesh_extractor,
                 "post": pipe.mesh_process.process_mesh, "dino": m["dinov2"].encode_images,
                 "g3d": AnimationPipeline.generate_3d_latents, "gma": AnimationPipeline.generate_mesh_animation}
    counts = {}

    def extract(lat):
        mesh = originals["s0_mesh"](lat)
        counts["before"] = {"vertices": len(mesh.vertices), "faces": len(mesh.faces)}
        return mesh

    def post(mesh, seed=None):
        out = originals["post"](mesh, seed=seed)
        counts["after"] = {"vertices": len(out.vertices), "faces": len(out.faces)}
        return out

    m["rmbg"].process_images = timer.wrap("background_removal", originals["rmbg"])
    pipe.image_process.process_images = timer.wrap("crop", originals["crop"])
    s0.image_encoder.encode_images = timer.wrap("stage0_dinov2", originals["s0_enc"])
    s0.denoise = timer.wrap("stage0_dit", originals["s0_denoise"])
    s0.mesh_extractor = timer.wrap("stage0_vae_dmc", extract)
    pipe.mesh_process.process_mesh = timer.wrap("postprocess", post)
    m["dinov2"].encode_images = timer.wrap("dinov2", originals["dino"])
    AnimationPipeline.generate_3d_latents = timer.wrap("stage1", originals["g3d"])
    AnimationPipeline.generate_mesh_animation = timer.wrap("stage2", originals["gma"])
    try:
        runs = []
        for i in range(calls + 1):                        # call 0 is the warm-up
            timer.t = {}
            inp = ActionMeshInput(frames(), torch.arange(16, dtype=torch.float32))
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            meshes = pipe(inp, seed=44)
            torch.cuda.synchronize()
            total = time.perf_counter() - t0
            if i:
                runs.append({**{k: timer.t.get(k, 0.0) for k in STAGES}, "total": total})
    finally:
        m["rmbg"].process_images, pipe.image_process.process_images = originals["rmbg"], originals["crop"]
        s0.image_encoder.encode_images, s0.denoise, s0.mesh_extractor = (originals["s0_enc"], originals["s0_denoise"],
                                                                         originals["s0_mesh"])
        m["dinov2"].encode_images = originals["dino"]
        AnimationPipeline.generate_3d_latents, AnimationPipeline.generate_mesh_animation = originals["g3d"], originals["gma"]
    return {"stage_0_steps": pipe.cfg.stage_0_steps, "stage_1_steps": pipe.cfg.stage_1_steps,
            "sec_per_video": {k: round(statistics.median(r[k] for r in runs), 4) for k in (*STAGES, "total")},
            "calls_total_s": [round(r["total"], 4) for r in runs], "anchor_mesh": counts, "output_meshes": len(meshes)}


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("video_e2e_bench: needs a CUDA device (H100); there is nothing to measure without one")
    card = gpu_card()
    m = build_models()
    from actionmesh_b200.preprocess import B200FramePreprocessor

    centre_field(m, B200FramePreprocessor().process_images(frames())[0], 100)
    res = {"metric": "video_to_4d_sec_per_video", "gpu": card,
           "inputs": "16 frames 512x512, uniform RGB seed 7, alpha disc r=180 (SURVEY 8(d)); seed 44",
           "weights": "random (seeded), full-size models; the Stage 0 surface is arbitrary",
           "timing": f"median of {args.calls} calls after 1 warm-up; host clock after a device synchronise",
           "configs": {c: run_config(m, c, args.calls) for c in CONFIGS}}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
