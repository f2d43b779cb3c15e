"""Write tests/golden/octree_fields.pt from the reference's OWN flash_extract_geometry and near-surface band.

    ACTIONMESH_REFERENCE=/path/to/actionmesh python tools/gen_octree_golden.py

Runs on the CPU with the stubs of tools/gen_triposg_vae_golden.py (the DiffDMC stub records the grid handed to it).
tests/golden/triposg_vae_tiny.pt is not touched.  Stored:
  * for the analytic fields of tests/geometry_exact.py substituted for the decoder (border_field, level_field and
    thin_field at octree_depth 8 and 9): the final logit grid as its finite cells in grid order
    (int32 linear indices, fp32 values): their count, SHA-256 digests of both arrays and the first entries in full;
  * for the adversarial grids geometry_exact.band_grid(n) of the small sides: the reference's band,
    extract_near_surface_volume_fn(grid, 0) + (|grid| < 0.95) > 0, as uint8, with the SHA-256 of the grid it was built from.
"""
from __future__ import annotations

import os
import sys
import time
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from oracle import reference_loader  # noqa: E402
import geometry_exact as gx  # noqa: E402
from gen_triposg_vae_golden import HEAD, _DecoderOutput, _install_stubs  # noqa: E402
from triposg_vae_ref import BOUNDS, sha256  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "octree_fields.pt")
FIELDS = (("border", 8), ("level", 8), ("thin", 8), ("border", 9), ("level", 9), ("thin", 9))
BAND_SIDES = (2, 3, 12, 13, 16)


def main():
    if not reference_loader.available():
        raise SystemExit(f"reference checkout not found at {reference_loader.REFERENCE_ROOT}")
    seen = _install_stubs()
    sys.path.insert(0, os.path.join(reference_loader.REFERENCE_ROOT, "third_party", "TripoSG"))
    from triposg.inference_utils import extract_near_surface_volume_fn, flash_extract_geometry

    torch.set_grad_enabled(False)
    bands = {}
    for n in BAND_SIDES:
        g = gx.band_grid(n)
        mask = extract_near_surface_volume_fn(g, 0.0)
        mask += g.abs() < 0.95                          # inference_utils.py:403
        bands[n] = {"sha256_grid": sha256(g), "mask": (mask > 0).to(torch.uint8)}
    fields = {}
    for name, depth in FIELDS:
        fn = getattr(gx, name + "_field")
        field_vae = types.SimpleNamespace(decoder=types.SimpleNamespace(set_topk=lambda *_: None),
                                          decode=lambda lat, q, fn=fn: _DecoderOutput(fn(q.reshape(-1, 3)).reshape(*q.shape[:-1], 1)))
        seen.clear()
        t0 = time.time()
        flash_extract_geometry(torch.zeros(1, 4, 64), field_vae, bounds=BOUNDS, octree_depth=depth)
        r = 2 ** depth
        while r >= 63:          # the `octree_resolution` left over from the ladder loop, a power of two: exact
            r //= 2
        grid = (-seen[0] * r).reshape(-1)
        idx = torch.nonzero(torch.isfinite(grid)).reshape(-1)
        idx, val = idx.to(torch.int32).contiguous(), grid[idx].contiguous()
        fields[(name, depth)] = {"side": int(seen[0].shape[0]), "count": idx.numel(), "sha256_index": sha256(idx),
                                 "sha256_values": sha256(val), "head_index": idx[:HEAD].clone(), "head_values": val[:HEAD].clone()}
        print(name, depth, seen[0].shape[0], idx.numel(), f"{time.time() - t0:.1f} s")
    torch.save({"bounds": BOUNDS, "fields": fields, "bands": bands}, GOLDEN)
    print(GOLDEN, os.path.getsize(GOLDEN))


if __name__ == "__main__":
    main()
