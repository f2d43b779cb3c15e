"""Regenerate tests/golden/triposg_vae_tiny.pt from the reference's OWN TripoSG VAE and flash_extract_geometry.

    ACTIONMESH_REFERENCE=/path/to/actionmesh python tools/gen_triposg_vae_golden.py

Needs a checkout of facebookresearch/actionmesh (third_party/TripoSG is imported unchanged on top of oracle/diffusers_shim.py).
`diso`, `skimage` and `omegaconf` are not needed on this path and are stubbed; the DiffDMC stub records the signed-distance
grid flash_extract_geometry hands to it and returns an empty mesh.  Stored:
  * a seeded tiny TripoSGVAEModel (width_decoder 256, 2 heads x 128, 2 layers, 2048 latent tokens): decode logits at 4096
    points;
  * for the analytic sphere and torus fields of tests/triposg_vae_ref.py substituted for the decoder: the final logit grid
    at octree_depth 7 and 8 as its finite cells in grid order (int32 linear indices, fp32 values): their count, SHA-256
    digests of both arrays and the first entries in full.
"""
from __future__ import annotations

import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import diffusers_shim, reference_loader  # noqa: E402
import triposg_vae_ref as ref  # noqa: E402
from triposg_vae_ref import sha256  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "triposg_vae_tiny.pt")
SEED, INPUT_SEED = 515, 9
HEAD = 2000   # leading entries of each sparse grid stored in full (for diagnosing a mismatch); the rest as digests


class _DecoderOutput:
    def __init__(self, sample):
        self.sample = sample


def _install_stubs():
    diffusers_shim.install()

    def mod(name, **attrs):
        m = sys.modules.get(name) or types.ModuleType(name)
        for k, v in attrs.items():
            setattr(m, k, v)
        sys.modules[name] = m
        return m

    mod("diffusers.models.autoencoders")
    mod("diffusers.models.autoencoders.vae", DecoderOutput=_DecoderOutput)
    mod("diffusers.models.modeling_outputs", AutoencoderKLOutput=type("AutoencoderKLOutput", (), {}))
    mod("diffusers.utils.accelerate_utils", apply_forward_hook=lambda f: f)
    sys.modules["diffusers.utils"].torch_utils.randn_tensor = torch.randn
    seen = []

    class DiffDMC(torch.nn.Module):
        def __init__(self, dtype=torch.float32):
            super().__init__()

        def forward(self, sdf, deform=None, return_quads=False, normalize=False):
            seen.append(sdf.clone())
            return torch.zeros(0, 3), torch.zeros(0, 3, dtype=torch.int64)

    mod("diso", DiffDMC=DiffDMC)
    mod("skimage", measure=types.SimpleNamespace())
    mod("omegaconf", DictConfig=dict, ListConfig=list)
    return seen


def main():
    if not reference_loader.available():
        raise SystemExit(f"reference checkout not found at {reference_loader.REFERENCE_ROOT}")
    seen = _install_stubs()
    sys.path.insert(0, os.path.join(reference_loader.REFERENCE_ROOT, "third_party", "TripoSG"))
    from triposg.inference_utils import flash_extract_geometry
    from triposg.models.autoencoders.autoencoder_kl_triposg import TripoSGVAEModel

    torch.set_grad_enabled(False)
    cfg = ref.TINY
    vae = TripoSGVAEModel(num_attention_heads=cfg["num_attention_heads"], width_decoder=cfg["width_decoder"],
                          num_layers_decoder=cfg["num_layers_decoder"], width_encoder=256, num_layers_encoder=1).eval()
    sd = ref.make_state_dict(cfg["width_decoder"], cfg["num_attention_heads"], cfg["num_layers_decoder"], seed=SEED)
    full = vae.state_dict()
    full.update(sd)
    vae.load_state_dict(full, strict=True)   # also pins the decoder-side key names
    g = torch.Generator().manual_seed(INPUT_SEED)
    z = torch.randn(1, 2048, 64, generator=g)
    pts = torch.rand(1, 4096, 3, generator=g) * 2.01 - 1.005
    logits = vae.decode(z, pts).sample

    # flash_extract_geometry with an analytic field in place of the decoder
    fields = {}
    for name, fn in (("sphere", ref.sphere), ("torus", ref.torus)):
        field_vae = types.SimpleNamespace(decoder=types.SimpleNamespace(set_topk=lambda *_: None),
                                          decode=lambda lat, q, fn=fn: _DecoderOutput(fn(q.reshape(-1, 3)).reshape(*q.shape[:-1], 1)))
        for depth in (7, 8):
            seen.clear()
            flash_extract_geometry(torch.zeros(1, 4, 64), field_vae, bounds=ref.BOUNDS, octree_depth=depth)
            r = 2 ** depth
            while r >= 63:          # the `octree_resolution` left over from the ladder loop, a power of two: exact
                r //= 2
            grid = (-seen[0] * r).reshape(-1)
            idx = torch.nonzero(torch.isfinite(grid)).reshape(-1)
            idx, val = idx.to(torch.int32).contiguous(), grid[idx].contiguous()
            fields[(name, depth)] = {"side": int(seen[0].shape[0]), "count": idx.numel(), "sha256_index": sha256(idx),
                                     "sha256_values": sha256(val), "head_index": idx[:HEAD].clone(), "head_values": val[:HEAD].clone()}
    torch.save({"config": cfg, "seed": SEED, "input_seed": INPUT_SEED, "z": z, "points": pts, "logits": logits,
                "bounds": ref.BOUNDS, "fields": fields}, GOLDEN)
    print(GOLDEN, os.path.getsize(GOLDEN))
    for k, v in fields.items():
        print(k, v["side"], v["count"])


if __name__ == "__main__":
    main()
