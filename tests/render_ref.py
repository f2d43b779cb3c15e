"""numpy float32 restatement of the normal renderer's contract (DESIGN.md §16), used by test_render_cpu.py and
test_render_gpu.py.  Not collected by pytest.

Every operation is a separate float32 numpy operation in the order DESIGN.md writes it, so the kernels in csrc/render.cu,
which round each operation on its own, must match it bit for bit.  The rasterizer is brute force over every face for each
sample, like PyTorch3D's naive path; it can be restricted to chosen samples so large meshes are checked at sampled pixels.
"""
from __future__ import annotations

import numpy as np

f32 = np.float32
EPS = f32(1e-8)


def camera_table(cams: dict) -> tuple[np.ndarray, float]:
    """{tag: (R, T, f)} -> ((C, 12) float32 = R row-major then T, f)."""
    table = np.stack([np.concatenate([R.reshape(-1), T]) for R, T, _ in cams.values()]).astype(f32)
    return table, next(iter(cams.values()))[2]


def transform(p: np.ndarray, cam: np.ndarray, t: np.ndarray) -> tuple:
    """Row vectors p (..., 3) times R plus t, each output ((x R0j + y R1j) + z R2j) + t_j."""
    R = cam[:9].reshape(3, 3)
    x, y, z = p[..., 0], p[..., 1], p[..., 2]
    return tuple(((x * R[0, j] + y * R[1, j]) + z * R[2, j]) + t[j] for j in range(3))


def project(verts: np.ndarray, cam: np.ndarray, focal: float) -> np.ndarray:
    """(V, 3) world -> (V, 3) = (f X / Z', f Y / Z', Z), Z' = sign(Z) max(|Z|, 1e-8)."""
    vx, vy, vz = transform(verts.astype(f32), cam, cam[9:12])
    az = np.where(np.abs(vz) > EPS, np.abs(vz), EPS)
    zd = np.where(vz < 0, -az, az)
    fo = f32(focal)
    return np.stack([(fo * vx) / zd, (fo * vy) / zd, vz], axis=-1).astype(f32)


def sample_ndc(idx, n2: int) -> np.ndarray:
    """1 - (2i + 1) / 2S."""
    return f32(1) - (2 * np.asarray(idx, dtype=np.int64) + 1).astype(f32) / f32(n2)


def edge(px, py, a, b):
    return (px - a[0]) * (b[1] - a[1]) - (py - a[1]) * (b[0] - a[0])


def barycentrics(v0, v1, v2, px, py):
    """(inside, (b0, b1, b2)) at the sample coordinates px, py: perspective-corrected, strictly inside, clipped."""
    den = edge(v2[0], v2[1], v0, v1) + EPS
    w0, w1, w2 = edge(px, py, v1, v2) / den, edge(px, py, v2, v0) / den, edge(px, py, v0, v1) / den
    t0, t1, t2 = (w0 * v1[2]) * v2[2], (v0[2] * w1) * v2[2], (v0[2] * v1[2]) * w2
    st = (t0 + t1) + t2
    dn = np.where(st > EPS, st, EPS)
    p0, p1, p2 = t0 / dn, t1 / dn, t2 / dn
    inside = (p0 > 0) & (p1 > 0) & (p2 > 0)
    c0, c1, c2 = np.maximum(p0, f32(0)), np.maximum(p1, f32(0)), np.maximum(p2, f32(0))
    sc = (c0 + c1) + c2
    dc = np.where(sc > f32(1e-5), sc, f32(1e-5))
    return inside, (c0 / dc, c1 / dc, c2 / dc)


def rasterize_ref(verts: np.ndarray, faces: np.ndarray, cams: np.ndarray, focal: float, S: int, rows=None, cols=None):
    """pix_to_face of every camera: (C, 2S, 2S) int32, or (C, K) at the samples rows[c], cols[c] (each (C, K))."""
    n2 = 2 * S
    out = []
    with np.errstate(all="ignore"):
        for c, cam in enumerate(cams):
            if rows is None:
                r, q = np.meshgrid(np.arange(n2), np.arange(n2), indexing="ij")
            else:
                r, q = np.asarray(rows[c]), np.asarray(cols[c])
            px, py = sample_ndc(q, n2), sample_ndc(r, n2)
            best = np.full(r.shape, np.inf, dtype=f32)
            idx = np.full(r.shape, -1, dtype=np.int32)
            pv = project(verts, cam, focal)
            for f, (a, b, d) in enumerate(faces):
                v0, v1, v2 = pv[a], pv[b], pv[d]
                if np.abs(edge(v0[0], v0[1], v1, v2)) <= EPS or (v0[2] < 0 and v1[2] < 0 and v2[2] < 0):
                    continue
                inside, (b0, b1, b2) = barycentrics(v0, v1, v2, px, py)
                pz = ((b0 * v0[2]) + (b1 * v1[2])) + (b2 * v2[2])
                hit = inside & (pz >= 0) & (pz < best)
                best[hit] = pz[hit]
                idx[hit] = f
            out.append(idx)
    return np.stack(out)


def vertex_normals_ref(verts: np.ndarray, faces: np.ndarray) -> np.ndarray:
    """Per vertex the sum of cross(v1 - v0, v2 - v0) over its faces in ascending face order, over max(|n|, 1e-6)."""
    v = verts.astype(f32)
    p0, p1, p2 = v[faces[:, 0]], v[faces[:, 1]], v[faces[:, 2]]
    a, b = p1 - p0, p2 - p0
    cr = np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                   a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], axis=1).astype(f32)
    n = np.zeros_like(v)
    for k in range(3):  # unbuffered, in order of occurrence: ascending face order per vertex (corners are distinct)
        np.add.at(n[:, k], faces.reshape(-1), np.repeat(cr[:, k], 3))
    length = np.sqrt((n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2])
    d = np.where(length > f32(1e-6), length, f32(1e-6))
    return (n / d[:, None]).astype(f32)


def shade_ref(verts, faces, normals, cams, focal, S, quad: np.ndarray, i, j) -> tuple[np.ndarray, np.ndarray]:
    """(mask uint8 (C, K), rgb uint8 (C, K, 3)) of output pixels (i[c], j[c]) given pix_to_face at their samples
    quad (C, K, 4) = (2i, 2j), (2i, 2j+1), (2i+1, 2j), (2i+1, 2j+1)."""
    n2 = 2 * S
    masks, rgbs = [], []
    with np.errstate(all="ignore"):
        for c, cam in enumerate(cams):
            q = quad[c]
            mask = (q >= 0).sum(axis=1).astype(f32) * f32(0.25)
            f = q[:, 0]
            nrm = np.zeros((len(f), 3), dtype=f32)
            hit = f >= 0
            if hit.any():
                pv = project(verts, cam, focal)
                fc = faces[f[hit]]
                v0, v1, v2 = (pv[fc[:, k]].T for k in range(3))
                _, (b0, b1, b2) = barycentrics(v0, v1, v2, sample_ndc(2 * np.asarray(j[c])[hit], n2),
                                               sample_ndc(2 * np.asarray(i[c])[hit], n2))
                a0, a1, a2 = (normals[fc[:, k]] for k in range(3))
                nrm[hit] = ((b0[:, None] * a0) + (b1[:, None] * a1)) + (b2[:, None] * a2)
            t = np.stack(transform(nrm, cam, cam[9:12] * f32(0.5)), axis=-1).astype(f32)
            length = np.sqrt((t[:, 0] * t[:, 0] + t[:, 1] * t[:, 1]) + t[:, 2] * t[:, 2])
            d = np.where(length > f32(1e-12), length, f32(1e-12))
            ch = np.clip((t / d[:, None] + f32(1)) * f32(0.5), f32(0), f32(1))
            rgb = (ch * mask[:, None] + (f32(1) - mask)[:, None]) * f32(255)
            masks.append((mask * f32(255)).astype(np.uint8))
            rgbs.append(rgb.astype(np.uint8))
    return np.stack(masks), np.stack(rgbs)


def render_ref(verts, faces, cams, focal, S) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Full restatement -> (pix_to_face (C, 2S, 2S), mask uint8 (C, S, S), rgb uint8 (C, S, S, 3))."""
    p2f = rasterize_ref(verts, faces, cams, focal, S)
    normals = vertex_normals_ref(verts, faces) if len(faces) else np.zeros_like(verts, dtype=f32)
    C = len(cams)
    i, j = np.meshgrid(np.arange(S), np.arange(S), indexing="ij")
    quad = np.stack([p2f[:, 0::2, 0::2], p2f[:, 0::2, 1::2], p2f[:, 1::2, 0::2], p2f[:, 1::2, 1::2]], axis=-1)
    mask, rgb = shade_ref(verts, faces, normals, cams, focal, S, quad.reshape(C, -1, 4),
                          np.broadcast_to(i.reshape(-1), (C, S * S)), np.broadcast_to(j.reshape(-1), (C, S * S)))
    return p2f, mask.reshape(C, S, S), rgb.reshape(C, S, S, 3)


def rasterize_pairs_ref(verts, faces, cam, focal, S, rows, cols, pair_sample, pair_face) -> np.ndarray:
    """pix_to_face (K,) at samples (rows, cols) of one camera, evaluating the contract only for the given (sample, face)
    pairs: every face that can cover a sample must appear with it (for large meshes, the faces whose projected box, widened
    by a few samples, holds the sample).  Same arithmetic as rasterize_ref, vectorized over pairs."""
    n2 = 2 * S
    pv = project(verts, cam, focal)
    fc = faces[pair_face]
    v0, v1, v2 = (pv[fc[:, k]].T for k in range(3))
    with np.errstate(all="ignore"):
        live = ~(np.abs(edge(v0[0], v0[1], v1, v2)) <= EPS) & ~((v0[2] < 0) & (v1[2] < 0) & (v2[2] < 0))
        inside, (b0, b1, b2) = barycentrics(v0, v1, v2, sample_ndc(np.asarray(cols)[pair_sample], n2),
                                            sample_ndc(np.asarray(rows)[pair_sample], n2))
        pz = ((b0 * v0[2]) + (b1 * v1[2])) + (b2 * v2[2])
    hit = live & inside & (pz >= 0)
    s, f, z = pair_sample[hit], pair_face[hit], pz[hit]
    order = np.lexsort((f, z, s))  # per sample: smallest depth, then lowest face
    s, f = s[order], f[order]
    first = np.ones(len(s), dtype=bool)
    first[1:] = s[1:] != s[:-1]
    out = np.full(len(rows), -1, dtype=np.int32)
    out[s[first]] = f[first]
    return out
