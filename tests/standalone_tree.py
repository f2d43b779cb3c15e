"""A tiny checkpoint tree in the reference's `pretrained_weights/` layout and key names (actionmesh/pipeline.py:66-83), from
seeded weights: safetensors plus config.json, preprocessor_config.json and scheduler_config.json.  RMBG has a fixed
architecture, so it is written at full size.  Used by tests/test_standalone_pipeline_gpu.py."""
from __future__ import annotations

import dataclasses
import json
import os

import numpy as np
import torch

N_TOKENS = 64          # Stage 0 / Stage I latent tokens of the tiny tree
DINO = dict(hidden_size=256, num_layers=2, num_heads=4)
DIT = dict(num_attention_heads=2, width=256, in_channels=64, num_layers=5, cross_attention_dim=256)
VAE = dict(width_decoder=256, num_attention_heads=2, num_layers_decoder=2, width_encoder=256, num_layers_encoder=2,
           embed_frequency=2)   # a low-frequency field: a few smooth blobs rather than a depth-9 foam
SHIFT = 3.0


def _save(sd: dict, path: str) -> None:
    from safetensors.torch import save_file

    os.makedirs(os.path.dirname(path), exist_ok=True)
    save_file({k: v.detach().to("cpu", torch.float32).contiguous() for k, v in sd.items()}, path)


def _json(obj: dict, path: str) -> None:
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "w") as f:
        json.dump(obj, f)


def write_dinov2(model_dir: str, feature_extractor_dir: str, crop: int, seed: int) -> None:
    """An HF Dinov2Model (config.json image_size 518: the position-embedding grid) and a BitImageProcessor cropping `crop`."""
    from actionmesh_b200.image_encoder import default_preprocessor
    from oracle import dinov2_oracle

    dinov2_oracle.make_model(DINO["hidden_size"], DINO["num_layers"], DINO["num_heads"], seed=seed).save_pretrained(model_dir)
    proc = default_preprocessor()
    proc.size = {"shortest_edge": max(256, crop)}
    proc.crop_size = {"height": crop, "width": crop}
    proc.save_pretrained(feature_extractor_dir)


def vae_state_dict(seed: int = 8) -> dict:
    import triposg_vae_encoder_ref as eref
    import triposg_vae_ref as ref

    sd = ref.make_state_dict(VAE["width_decoder"], VAE["num_attention_heads"], VAE["num_layers_decoder"],
                             embed_frequency=VAE["embed_frequency"], seed=seed)
    sd.update(eref.make_encoder_state_dict(VAE["width_encoder"], VAE["num_attention_heads"], VAE["num_layers_encoder"],
                                           embed_frequency=VAE["embed_frequency"], seed=seed + 1))
    return sd


def write_vae(triposg_dir: str, sd: dict) -> None:
    _json(VAE, os.path.join(triposg_dir, "vae", "config.json"))
    _save(sd, os.path.join(triposg_dir, "vae", "diffusion_pytorch_model.safetensors"))


def write_triposg(triposg_dir: str, crop: int = 224, seed: int = 4242) -> None:
    from actionmesh_b200.blocks import TRIPOSG_BLOCK_KEYS, remap_block_keys
    from oracle import synth

    class Cfg:
        mlp_ratio = 4.0
        in_channels, num_layers, num_attention_heads = DIT["in_channels"], DIT["num_layers"], DIT["num_attention_heads"]
        width, cross_attention_dim = DIT["width"], DIT["cross_attention_dim"]

    sd = remap_block_keys(synth.make_state_dict(Cfg(), seed), [(b, a) for a, b in TRIPOSG_BLOCK_KEYS])  # TripoSG key names
    _json({"_class_name": "TripoSGDiTModel", **DIT, "use_cross_attention_2": False},
          os.path.join(triposg_dir, "transformer", "config.json"))
    _save(sd, os.path.join(triposg_dir, "transformer", "diffusion_pytorch_model.safetensors"))
    write_vae(triposg_dir, vae_state_dict())
    write_dinov2(os.path.join(triposg_dir, "image_encoder_dinov2"), os.path.join(triposg_dir, "feature_extractor_dinov2"),
                 crop, seed=7)
    _json({"_class_name": "RectifiedFlowScheduler", "num_train_timesteps": 1000, "shift": SHIFT,
           "use_dynamic_shifting": False}, os.path.join(triposg_dir, "scheduler", "scheduler_config.json"))


def write_tree(root: str, triposg_crop: int = 224) -> str:
    """The four directories of `pretrained_weights/`: TripoSG, dinov2, RMBG, ActionMesh."""
    import rmbg_ref

    from actionmesh_b200.autoencoder import AutoencoderConfig
    from actionmesh_b200.denoiser import DenoiserConfig
    from oracle import autoencoder_oracle as ao
    from oracle import synth

    write_triposg(os.path.join(root, "TripoSG"), triposg_crop)
    dino = os.path.join(root, "dinov2")
    write_dinov2(dino, dino, 224, seed=5)
    _save(rmbg_ref.make_state_dict(0, device="cuda"), os.path.join(root, "RMBG", "model.safetensors"))
    dcfg = DenoiserConfig(num_tokens_nominal=N_TOKENS, num_layers=3, num_attention_heads=2, width=256,
                          cross_attention_dim=DINO["hidden_size"], in_channels=64, inflated_layers=(0, 1, 2))
    _json(dataclasses.asdict(dcfg), os.path.join(root, "ActionMesh", "denoiser", "config.json"))
    _save(synth.make_state_dict(dcfg, 17), os.path.join(root, "ActionMesh", "denoiser", "model.safetensors"))
    acfg = AutoencoderConfig(width=256, num_layers=2, num_attention_heads=2, temporal_context_size=16)
    _json(dataclasses.asdict(acfg), os.path.join(root, "ActionMesh", "autoencoder", "config.json"))
    _save(ao.make_autoencoder_state_dict(ao.AutoencoderConfig(width=256, num_layers=2, num_attention_heads=2), 99),
          os.path.join(root, "ActionMesh", "autoencoder", "model.safetensors"))
    return root


def centre_vae_field(root: str, latents: list) -> dict:
    """Shift the VAE's proj_out bias so that the decoded field of `latents` is zero at its median over a 64^3 grid: the
    random decoder then has a surface (half of the box inside) instead of none.  Returns the VAE's state dict."""
    import triposg_vae_ref as ref

    sd = vae_state_dict()
    a = torch.linspace(-1.005, 1.005, 64)
    xyz = torch.stack(torch.meshgrid(a, a, a, indexing="ij"), -1).reshape(1, -1, 3).cuda()
    vals = torch.cat([ref.decode_fp32(sd, lat, xyz, VAE["num_attention_heads"], VAE["num_layers_decoder"],
                                      embed_frequency=VAE["embed_frequency"]).reshape(-1) for lat in latents])
    sd["decoder.proj_out.bias"] = sd["decoder.proj_out.bias"] + vals.median().cpu()
    write_vae(os.path.join(root, "TripoSG"), sd)
    return sd


def rgba_frames(n: int = 16, size: int = 128, seed: int = 3) -> list:
    """`n` seeded random RGB frames with an alpha disc (a valid alpha: background removal passes them through)."""
    from PIL import Image

    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:size, 0:size]
    out = []
    for i in range(n):
        rgba = rng.integers(0, 255, (size, size, 4), dtype=np.uint8)
        cx, cy = size / 2 + 4 * np.sin(i / 3), size / 2 + 3 * np.cos(i / 4)
        rgba[..., 3] = np.where((x - cx) ** 2 + (y - cy) ** 2 < (0.3 * size) ** 2, 255, 0)
        out.append(Image.fromarray(rgba, "RGBA"))
    return out
