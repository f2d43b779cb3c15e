"""numpy float32 restatement of per-face material shading (DESIGN.md §16, "Texture shading", shading records), used by
test_multi_material_gpu.py.  Not collected by pytest.

Each covered sample shades with its face's record exactly as render_texture_ref.py shades a sample with one texture: the
record's chain sets the level of detail from its own level 0 size.  The four-sample mean and truncation are the same.
"""
from __future__ import annotations

import numpy as np

import render_texture_ref as tr

f32 = np.float32


def shade_materials_ref(verts, faces, normals, uv, cams, focal, S, pix_to_face, face_record, records) -> np.ndarray:
    """The cells (C, S, S, 3) uint8 of pix_to_face (C, 2S, 2S) when face f shades with records[face_record[f]], each record
    (chain: a list of levels as `tr.mip_chain` gives it, or None; (mag, min, wrap_s, wrap_t); base colour RGB)."""
    n2 = 2 * S
    face_record = np.asarray(face_record)
    out = []
    r, c = np.meshgrid(np.arange(n2), np.arange(n2), indexing="ij")
    for view, cam in enumerate(cams):
        p2f = pix_to_face[view]
        col = np.ones((n2, n2, 3), dtype=f32)
        hit = p2f >= 0
        rec = np.full(p2f.shape, -1)
        rec[hit] = face_record[p2f[hit]]
        for k in np.unique(rec[hit]):
            sel = rec == k
            chain, sampler, base = records[k]
            col[sel] = tr.shade_samples_ref(verts, faces, normals, uv, cam, focal, S, r[sel], c[sel], p2f[sel], chain,
                                            sampler, base)
        q = col.reshape(S, 2, S, 2, 3)
        acc = ((q[:, 0, :, 0] + q[:, 0, :, 1]) + q[:, 1, :, 0]) + q[:, 1, :, 1]
        out.append((np.clip(acc * f32(0.25), f32(0), f32(1)) * f32(255)).astype(np.uint8))
    return np.stack(out)
