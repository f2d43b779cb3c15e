"""numpy float32 restatement of the texture modality's contract (DESIGN.md §16, "Texture shading"), used by
test_render_texture_cpu.py and test_render_texture_gpu.py.  Not collected by pytest.

Every operation is a separate float32 numpy operation in the order DESIGN.md writes it, so `shade_texture_kernel` in
csrc/render.cu, which rounds each operation on its own, must match it bit for bit.  Projection and barycentrics come from
render_ref.py unchanged.
"""
from __future__ import annotations

import numpy as np

from render_ref import barycentrics, edge, project, sample_ndc

f32 = np.float32
NEAREST, LINEAR = 9728, 9729
NEAREST_MIPMAP_NEAREST, LINEAR_MIPMAP_NEAREST, NEAREST_MIPMAP_LINEAR, LINEAR_MIPMAP_LINEAR = 9984, 9985, 9986, 9987
REPEAT, CLAMP_TO_EDGE, MIRRORED_REPEAT = 10497, 33071, 33648
MIN_FILTERS = (NEAREST, LINEAR, NEAREST_MIPMAP_NEAREST, LINEAR_MIPMAP_NEAREST, NEAREST_MIPMAP_LINEAR, LINEAR_MIPMAP_LINEAR)
WRAPS = (REPEAT, CLAMP_TO_EDGE, MIRRORED_REPEAT)
UV_LIMIT = f32(32768)


def mip_chain(img: np.ndarray) -> list[np.ndarray]:
    """(h, w, 3) uint8 -> every level down to 1 x 1: level l + 1 is (max(1, h >> 1), max(1, w >> 1)) and each texel is
    floor((a + b + c + d + 2) / 4) over level-l texels (min(2x + dx, w - 1), min(2y + dy, h - 1))."""
    levels = [np.asarray(img, dtype=np.uint8)]
    while levels[-1].shape[:2] != (1, 1):
        a = levels[-1].astype(np.int32)
        h, w = a.shape[:2]
        ys, xs = np.arange(max(1, h >> 1)), np.arange(max(1, w >> 1))
        y0, y1 = np.minimum(2 * ys, h - 1), np.minimum(2 * ys + 1, h - 1)
        x0, x1 = np.minimum(2 * xs, w - 1), np.minimum(2 * xs + 1, w - 1)
        s = a[y0][:, x0] + a[y0][:, x1] + a[y1][:, x0] + a[y1][:, x1] + 2
        levels.append((s // 4).astype(np.uint8))
    return levels


def wrap(i: np.ndarray, n: int, mode: int) -> np.ndarray:
    """Integer texel index i wrapped into [0, n)."""
    i = np.asarray(i, dtype=np.int64)
    if mode == CLAMP_TO_EDGE:
        return np.clip(i, 0, n - 1)
    if mode == MIRRORED_REPEAT:
        m = np.mod(i, 2 * n)
        return np.where(m < n, m, 2 * n - 1 - m)
    assert mode == REPEAT
    return np.mod(i, n)


def sample_level(level: np.ndarray, u, v, linear: bool, wrap_s: int = REPEAT, wrap_t: int = REPEAT) -> np.ndarray:
    """Filtered RGB (K, 3) float32 in 0..255 of one level at (u, v) (each (K,)): NEAREST texel (floor(u w), floor(v h)), or
    LINEAR around (u w - 1/2, v h - 1/2); u and v are first clamped to +-2^15."""
    h, w = level.shape[:2]
    u = np.minimum(np.maximum(np.asarray(u, dtype=f32), -UV_LIMIT), UV_LIMIT)
    v = np.minimum(np.maximum(np.asarray(v, dtype=f32), -UV_LIMIT), UV_LIMIT)
    tex = lambda x, y: level[wrap(y, h, wrap_t), wrap(x, w, wrap_s)].astype(f32)  # noqa: E731
    if not linear:
        return tex(np.floor(u * f32(w)).astype(np.int64), np.floor(v * f32(h)).astype(np.int64))
    x, y = u * f32(w) - f32(0.5), v * f32(h) - f32(0.5)
    xf, yf = np.floor(x), np.floor(y)
    fx, fy = (x - xf)[:, None], (y - yf)[:, None]
    gx, gy = f32(1) - fx, f32(1) - fy
    xi, yi = xf.astype(np.int64), yf.astype(np.int64)
    t00, t10, t01, t11 = tex(xi, yi), tex(xi + 1, yi), tex(xi, yi + 1), tex(xi + 1, yi + 1)
    return ((t00 * gx + t10 * fx) * gy) + ((t01 * gx + t11 * fx) * fy)


def level_of_detail(a_t, a_s, positive_depth, n_levels: int, mag_filter: int, min_filter: int):
    """(level (K,), filter (K,)) per (face, view): magnified (A_t <= A_s) or a depth <= 0 -> level 0 and mag_filter;
    otherwise min_filter, and for a mip mode the smallest L with A_t <= ldexp(A_s, 2L), clamped to the last level."""
    a_t, a_s = np.asarray(a_t, dtype=f32), np.asarray(a_s, dtype=f32)
    minified = np.asarray(positive_depth) & ~(a_t <= a_s)
    level = np.zeros(a_t.shape, dtype=np.int64)
    if min_filter >= NEAREST_MIPMAP_NEAREST:
        with np.errstate(over="ignore"):
            for L in range(n_levels - 1, -1, -1):  # the smallest L that holds wins
                level = np.where(a_t <= np.ldexp(a_s, 2 * L).astype(f32), L, level)
            level = np.where(a_t <= np.ldexp(a_s, 2 * (n_levels - 1)).astype(f32), level, n_levels - 1)
        level = np.where(minified, level, 0)
    return level, np.where(minified, min_filter, mag_filter)


def is_linear(filter_):
    return np.isin(filter_, (LINEAR, LINEAR_MIPMAP_NEAREST, LINEAR_MIPMAP_LINEAR))


def shade_samples_ref(verts, faces, normals, uv, cam, focal, S, rows, cols, f, levels=None, sampler=None,
                      base=(1.0, 1.0, 1.0)) -> np.ndarray:
    """Colour (K, 3) float32 of the samples (rows, cols) of one view covered by faces f (all >= 0)."""
    n2 = 2 * S
    mag, mn, ws, wt = sampler or (LINEAR, LINEAR_MIPMAP_NEAREST, REPEAT, REPEAT)
    base = np.asarray(base, dtype=f32)
    with np.errstate(all="ignore"):
        pv = project(verts, cam, focal)
        fc = faces[f]
        v0, v1, v2 = (pv[fc[:, k]].T for k in range(3))
        _, (b0, b1, b2) = barycentrics(v0, v1, v2, sample_ndc(cols, n2), sample_ndc(rows, n2))
        a0, a1, a2 = (normals[fc[:, k]] for k in range(3))
        n = ((b0[:, None] * a0) + (b1[:, None] * a1)) + (b2[:, None] * a2)
        R = cam[:9].reshape(3, 3)
        vx, vy, vz = (((n[:, 0] * R[0, j]) + (n[:, 1] * R[1, j])) + (n[:, 2] * R[2, j]) for j in range(3))
        length = np.sqrt((vx * vx + vy * vy) + vz * vz)
        d = np.where(length > f32(1e-12), length, f32(1e-12))
        shade = f32(0.35) + f32(0.65) * np.abs(vz / d)
        col = np.broadcast_to(base, (len(f), 3)).astype(f32)
        if levels is not None:
            t0, t1, t2 = (uv[fc[:, k]] for k in range(3))
            u = ((b0 * t0[:, 0]) + (b1 * t1[:, 0])) + (b2 * t2[:, 0])
            v = ((b0 * t0[:, 1]) + (b1 * t1[:, 1])) + (b2 * t2[:, 1])
            a_s = (f32(0.5) * np.abs(edge(v0[0], v0[1], v1, v2))) * f32(S * S)
            a_t = (f32(0.5) * np.abs(edge(t0[:, 0], t0[:, 1], t1.T, t2.T))) * f32(levels[0].shape[0] * levels[0].shape[1])
            pos = (v0[2] > 0) & (v1[2] > 0) & (v2[2] > 0)
            level, filt = level_of_detail(a_t, a_s, pos, len(levels), mag, mn)
            tex = np.zeros((len(f), 3), dtype=f32)
            lin = is_linear(filt)
            for L in np.unique(level):
                for linear in (False, True):
                    sel = (level == L) & (lin == linear)
                    if sel.any():
                        tex[sel] = sample_level(levels[L], u[sel], v[sel], linear, ws, wt)
            col = base * (tex / f32(255))
        return (col * shade[:, None]).astype(f32)


def shade_texture_ref(verts, faces, normals, uv, cams, focal, S, pix_to_face, levels=None, sampler=None,
                      base=(1.0, 1.0, 1.0)) -> np.ndarray:
    """The texture modality's cells (C, S, S, 3) uint8 from pix_to_face (C, 2S, 2S): each pixel the mean of its samples
    (2i + dy, 2j + dx) in the order (0,0), (0,1), (1,0), (1,1), a sample without a face being white."""
    n2 = 2 * S
    out = []
    r, c = np.meshgrid(np.arange(n2), np.arange(n2), indexing="ij")
    for view, cam in enumerate(cams):
        p2f = pix_to_face[view]
        col = np.ones((n2, n2, 3), dtype=f32)
        hit = p2f >= 0
        if hit.any():
            col[hit] = shade_samples_ref(verts, faces, normals, uv, cam, focal, S, r[hit], c[hit], p2f[hit], levels,
                                         sampler, base)
        q = col.reshape(S, 2, S, 2, 3)
        acc = ((q[:, 0, :, 0] + q[:, 0, :, 1]) + q[:, 1, :, 0]) + q[:, 1, :, 1]
        out.append((np.clip(acc * f32(0.25), f32(0), f32(1)) * f32(255)).astype(np.uint8))
    return np.stack(out)
