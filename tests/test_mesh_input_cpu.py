"""Host preparation of a user-supplied anchor mesh (actionmesh_b200/mesh_input.py): merge and clean, normalization round trip
and area-weighted surface sampling."""
import numpy as np
import pytest
import torch
from scipy import stats

from actionmesh_b200.mesh_input import (NormalizationParams, denormalize_mesh, face_normals, merge_and_clean_mesh,
                                        normalize_mesh, sample_surface)


class _Mesh:
    def __init__(self, vertices, faces):
        self.vertices, self.faces = vertices, faces


_CUBE_FACES = [  # 6 quads as (corner indices), each split in two triangles
    (0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]


def split_seam_cube(offset=(0.3, -1.2, 5.0), size=2.5):
    """A cube whose 6 faces each own their 4 corners: 24 vertices (8 distinct positions), 12 triangles."""
    corners = np.array([[(i >> 2) & 1, (i >> 1) & 1, i & 1] for i in range(8)], dtype=np.float64) * size + np.array(offset)
    verts, faces = [], []
    for quad in _CUBE_FACES:
        base = len(verts)
        verts.extend(corners[list(quad)])
        faces.extend([(base, base + 1, base + 2), (base, base + 2, base + 3)])
    return np.array(verts), np.array(faces, dtype=np.int64)


def test_merge_split_seams_round_trip():
    v, f = split_seam_cube()
    mesh = _Mesh(v.copy(), f.copy())
    vmap, pre_faces = merge_and_clean_mesh(mesh)
    assert len(mesh.vertices) == 8 and len(mesh.faces) == 12
    assert np.array_equal(mesh.vertices[vmap], v)
    assert np.array_equal(pre_faces, f)
    assert np.array_equal(vmap[f], mesh.faces)              # same triangles on the merged vertices
    assert len(np.unique(vmap)) == 8


def test_merge_drops_degenerate_duplicate_faces_and_unreferenced_vertices():
    v, f = split_seam_cube()
    v = np.concatenate([v, v[:1] + 1e-10])                  # a copy of vertex 0 within the rounding: merged
    extra = np.array([[0, 24, 1],                            # degenerate once 24 merges into 0
                      [2, 1, 0],                             # duplicate of face 0 as a sorted triple
                      [5, 6, 4]], dtype=np.int64)            # duplicate of face 2 (4, 5, 6), rotated
    f2 = np.concatenate([f, extra])
    mesh = _Mesh(v.copy(), f2.copy())
    vmap, pre_faces = merge_and_clean_mesh(mesh)
    assert np.array_equal(pre_faces, f2)
    assert len(mesh.vertices) == 8
    # every remaining face is non-degenerate and unique as a sorted triple
    faces = np.asarray(mesh.faces)
    assert (faces[:, 0] != faces[:, 1]).all() and (faces[:, 1] != faces[:, 2]).all() and (faces[:, 0] != faces[:, 2]).all()
    assert len(np.unique(np.sort(faces, axis=1), axis=0)) == len(faces)
    assert len(faces) == 12                                  # the cube's 12 triangles, the extras gone


def test_merge_keeps_first_occurrence_order():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 0, 0]], dtype=np.float64)
    mesh = _Mesh(v, np.array([[2, 1, 0], [2, 3, 0]]))
    vmap, _ = merge_and_clean_mesh(mesh)
    assert vmap.tolist() == [0, 1, 2, 1]
    assert np.asarray(mesh.faces).tolist() == [[2, 1, 0]]


def test_normalize_round_trip_float64():
    rng = np.random.default_rng(1)
    v = rng.normal(size=(500, 3)) * np.array([3.0, 0.5, 1.0]) + np.array([10.0, -4.0, 2.0])
    mesh = _Mesh(v.copy(), np.zeros((0, 3), dtype=np.int64))
    _, params = normalize_mesh(mesh)
    nv = np.asarray(mesh.vertices)
    assert isinstance(params, NormalizationParams)
    ext = nv.max(axis=0) - nv.min(axis=0)
    assert abs(ext.max() - 2.0) < 1e-12 and np.allclose((nv.max(axis=0) + nv.min(axis=0)) / 2, 0, atol=1e-12)
    denormalize_mesh(mesh, params)
    assert np.abs(np.asarray(mesh.vertices) - v).max() <= 1e-12


def _uneven_mesh():
    """Triangles of very different areas, not sharing vertices."""
    rng = np.random.default_rng(3)
    verts, faces = [], []
    for s in (0.1, 0.5, 1.0, 2.0, 3.0, 0.3):
        tri = rng.normal(size=(3, 3)) * s
        faces.append(list(range(len(verts), len(verts) + 3)))
        verts.extend(tri)
    return np.array(verts), np.array(faces, dtype=np.int64)


def test_sample_surface_points_lie_in_their_faces_with_unit_normals():
    v, f = _uneven_mesh()
    mesh = _Mesh(v, f)
    s = sample_surface(mesh, 4000, seed=7)
    assert s.shape == (1, 4000, 6) and s.dtype == torch.float64
    pts, nrm = s[0, :, :3].numpy(), s[0, :, 3:].numpy()
    fn = face_normals(v, f)
    # recover each point's face from its normal, then its barycentric coordinates
    face = np.array([np.argmin(np.linalg.norm(fn - n, axis=1)) for n in nrm])
    assert np.allclose(nrm, fn[face]) and np.allclose(np.linalg.norm(nrm, axis=1), 1.0)
    a, b, c = v[f[face, 0]], v[f[face, 1]], v[f[face, 2]]
    m = np.stack([b - a, c - a], axis=-1)
    uv = np.array([np.linalg.lstsq(mi, p - ai, rcond=None)[0] for mi, p, ai in zip(m, pts, a)])
    assert np.allclose(np.einsum("nij,nj->ni", m, uv) + a, pts, atol=1e-9)   # in the face's plane
    assert (uv >= -1e-9).all() and (uv.sum(axis=1) <= 1 + 1e-9).all()


def test_sample_surface_is_seeded():
    v, f = _uneven_mesh()
    a = sample_surface(_Mesh(v, f), 1000, seed=44)
    b = sample_surface(_Mesh(v, f), 1000, seed=44)
    c = sample_surface(_Mesh(v, f), 1000, seed=45)
    assert torch.equal(a, b) and not torch.equal(a, c)
    assert sample_surface(_Mesh(v, f), 10, seed=1, with_normals=False, dtype=torch.float32).shape == (1, 10, 3)


def test_sample_surface_face_counts_follow_areas():
    v, f = _uneven_mesh()
    n = 20000
    s = sample_surface(_Mesh(v, f), n, seed=11)
    fn = face_normals(v, f)
    face = np.array([np.argmin(np.linalg.norm(fn - x, axis=1)) for x in s[0, :, 3:].numpy()])
    area = 0.5 * np.linalg.norm(np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]]), axis=1)
    counts = np.bincount(face, minlength=len(f))
    _, p = stats.chisquare(counts, area / area.sum() * n)
    assert p > 1e-3, (counts, area / area.sum() * n)


@pytest.mark.parametrize("center", [True, False])
def test_normalize_without_center(center):
    v = np.array([[1.0, 2.0, 3.0], [3.0, 2.5, 3.5]])
    mesh, params = normalize_mesh(_Mesh(v.copy(), np.zeros((0, 3), dtype=np.int64)), center=center)
    assert (params.bbox_center is None) != center
    denormalize_mesh(mesh, params)
    assert np.allclose(mesh.vertices, v, atol=1e-12)
