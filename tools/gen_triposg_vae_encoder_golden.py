"""Regenerate tests/golden/triposg_vae_encoder_tiny.pt from the reference's OWN TripoSG VAE encoder.

    ACTIONMESH_REFERENCE=/path/to/actionmesh python tools/gen_triposg_vae_encoder_golden.py

Needs a checkout of facebookresearch/actionmesh: `TripoSGVAE` (actionmesh/external/triposg.py) and third_party/TripoSG are
imported unchanged on top of oracle/diffusers_shim.py.  pytorch3d is not needed: `sample_farthest_points` is stubbed with the
numpy FPS restatement of tests/triposg_vae_encoder_ref.py started at a recorded index (so is fpsample's,
which the reference calls for CPU tensors), `masked_gather` with a gather, and `randn_tensor` with a seeded torch.randn whose draw (eps) is recorded.  Modules off this path (trimesh, the TripoSG image
pipeline, diso, skimage, omegaconf) are stubbed.  Stored for a seeded tiny TripoSGVAEModel (width_encoder 256, 4 heads x 64,
2 layers; 4096 surface points, num_tokens 256): the surface, seed, FPS start and indices, the `quant` output of `_encode`,
and the latent of `encode_to_latent` with its eps.
"""
from __future__ import annotations

import functools
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from oracle import reference_loader  # noqa: E402
import triposg_vae_encoder_ref as ref  # noqa: E402
from gen_triposg_vae_golden import _install_stubs  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "triposg_vae_encoder_tiny.pt")
SEED, INPUT_SEED, SUBSET_SEED, START, EPS_SEED = 616, 10, 44, 123, 5
N_SURFACE, NUM_TOKENS = 4096, 256


def _mod(name, **attrs):
    m = sys.modules.get(name) or types.ModuleType(name)
    for k, v in attrs.items():
        setattr(m, k, v)
    sys.modules[name] = m
    return m


def main():
    if not reference_loader.available():
        raise SystemExit(f"reference checkout not found at {reference_loader.REFERENCE_ROOT}")
    _install_stubs()
    seen = {}

    def sample_farthest_points(points, K, random_start_point=True):
        assert random_start_point and points.shape[0] == 1
        idx = torch.from_numpy(ref.fps_numpy(points[0].numpy(), K, START))[None]
        seen["fps_points"], seen["fps_index"] = points.clone(), idx
        return points[:, idx[0]], idx

    def bucket_fps_kdline_sampling(points, n_samples, level, start_idx=None):
        """the CPU branch of _farthest_point_sample (pointcloud_sampling.py:64-86): start_idx None = random start"""
        assert start_idx is None
        idx = ref.fps_numpy(np.asarray(points), n_samples, START)
        seen["fps_points"], seen["fps_index"] = torch.as_tensor(np.asarray(points))[None].clone(), torch.from_numpy(idx)[None]
        return idx

    def randn_tensor(shape, generator=None, device=None, dtype=None):
        eps = torch.randn(shape, generator=torch.Generator().manual_seed(EPS_SEED), dtype=dtype)
        seen["eps"] = eps.clone()
        return eps

    _mod("pytorch3d")
    _mod("pytorch3d.ops", sample_farthest_points=sample_farthest_points)
    _mod("pytorch3d.ops.utils", masked_gather=lambda pts, idx: torch.stack([p[i] for p, i in zip(pts, idx)]))
    _mod("fpsample", fpsample=types.SimpleNamespace(bucket_fps_kdline_sampling=bucket_fps_kdline_sampling))
    sys.modules["diffusers.utils"].torch_utils.randn_tensor = randn_tensor
    _mod("diffusers.models.modeling_outputs", AutoencoderKLOutput=types.SimpleNamespace)
    _mod("trimesh", Trimesh=type("Trimesh", (), {}))
    _mod("diffusers.image_processor", PipelineImageInput=object)
    _mod("triposg.pipelines")
    _mod("triposg.pipelines.pipeline_triposg", TripoSGPipeline=type("TripoSGPipeline", (), {}))
    sys.path.insert(0, os.path.join(reference_loader.REFERENCE_ROOT, "third_party", "TripoSG"))
    sys.path.insert(0, reference_loader.REFERENCE_ROOT)
    from actionmesh.external.triposg import TripoSGVAE

    torch.set_grad_enabled(False)
    cfg = ref.TINY
    torch.manual_seed(SEED)
    vae = TripoSGVAE(num_attention_heads=cfg["num_attention_heads"], width_encoder=cfg["width_encoder"],
                     num_layers_encoder=cfg["num_layers_encoder"], width_decoder=cfg["width_decoder"],
                     num_layers_decoder=cfg["num_layers_decoder"]).eval()
    sd = ref.make_encoder_state_dict(cfg["width_encoder"], cfg["num_attention_heads"], cfg["num_layers_encoder"], seed=SEED)
    full = vae.state_dict()
    assert set(sd) <= set(full), sorted(set(sd) - set(full))   # pins the encoder-side key names
    full.update(sd)
    vae.load_state_dict(full, strict=True)
    vae.device, vae.dtype = torch.device("cpu"), torch.float32   # ModelMixin properties the diffusers stand-in lacks
    surface = ref.sphere_surface(N_SURFACE, INPUT_SEED)

    quant = vae._encode(surface, num_tokens=NUM_TOKENS, seed=SUBSET_SEED)
    subset = np.random.default_rng(SUBSET_SEED).choice(N_SURFACE, 4 * NUM_TOKENS, replace=4 * NUM_TOKENS > N_SURFACE)
    assert torch.equal(seen["fps_points"][0], surface[0, torch.from_numpy(subset), :3])
    fps_index = seen["fps_index"][0]
    vae._encode = functools.partial(TripoSGVAE._encode, vae, num_tokens=NUM_TOKENS, seed=SUBSET_SEED)
    latent = vae.encode_to_latent(surface)
    torch.save({"config": cfg, "seed": SEED, "surface": surface, "subset_seed": SUBSET_SEED, "subset": torch.from_numpy(subset),
                "num_tokens": NUM_TOKENS, "fps_start": START, "fps_index": fps_index, "quant": quant, "eps": seen["eps"],
                "latent": latent}, GOLDEN)
    print(GOLDEN, os.path.getsize(GOLDEN), tuple(quant.shape), tuple(latent.shape))


if __name__ == "__main__":
    main()
