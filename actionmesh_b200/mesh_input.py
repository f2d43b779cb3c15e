"""Host preparation of a user-supplied anchor mesh for the {video + 3D mesh} -> 4D pipeline (numpy + scipy).

Same signatures and return values as the reference's actionmesh/preprocessing/mesh_processor.py:
  merge_and_clean_mesh   :37-82   merge seam duplicates, drop degenerate / duplicate faces and unreferenced vertices
                                  (the rules are `clean_topology`, which B200MeshPostprocessor shares)
  normalize_mesh         :177-212 centre the bounding box, scale by 2 / max extent
  denormalize_mesh       :215-237 the inverse
  sample_surface         :245-285 area-weighted surface samples with their face normals -> (1, n, 3|6) tensor
They take a `trimesh.Trimesh` or any object with `.vertices` / `.faces` arrays and modify it in place like the reference (by
assigning `.vertices` / `.faces`).  These run once per video over at most 16384 samples, so they stay on the CPU, as in the
reference; the reference calls into trimesh for the merge and sampling rules, which are restated in the docstrings below.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch
from scipy.spatial import cKDTree

MERGE_DECIMALS = 8


def _arrays(mesh) -> tuple[np.ndarray, np.ndarray]:
    return np.asarray(mesh.vertices, dtype=np.float64), np.asarray(mesh.faces, dtype=np.int64).reshape(-1, 3)


def clean_topology(verts: np.ndarray, faces: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """The reference's topology clean-up (trimesh merge_vertices, remove_degenerate_faces, remove_duplicate_faces,
    remove_unreferenced_vertices) on (V, 3) float64 vertices and (F, 3) int64 faces -> new (vertices, faces).  Rules, in order:
      1. vertices whose coordinates are equal after rounding to 8 decimals become one vertex, placed at the first of them;
         the merged vertices keep the order of their first occurrence;
      2. faces that use a vertex twice are dropped;
      3. faces that repeat an earlier face as a sorted index triple are dropped (the first one is kept);
      4. vertices no face references are dropped."""
    _, first, inverse = np.unique(np.round(verts, MERGE_DECIMALS) + 0.0, axis=0, return_index=True, return_inverse=True)
    order = np.argsort(first, kind="stable")           # merged vertices in order of first occurrence
    rank = np.empty_like(order)
    rank[order] = np.arange(len(order))
    verts = verts[first[order]]
    faces = rank[inverse.reshape(-1)][faces]

    faces = faces[(faces[:, 0] != faces[:, 1]) & (faces[:, 1] != faces[:, 2]) & (faces[:, 0] != faces[:, 2])]
    _, keep = np.unique(np.sort(faces, axis=1), axis=0, return_index=True)
    faces = faces[np.sort(keep)]

    used = np.zeros(len(verts), dtype=bool)
    used[faces.reshape(-1)] = True
    remap = np.cumsum(used) - 1
    return verts[used], remap[faces]


def merge_and_clean_mesh(mesh) -> tuple[np.ndarray, np.ndarray]:
    """Merge duplicate vertices and clean the topology of `mesh` in place (`clean_topology`'s rules) ->
    (vertex_merge_map, pre_merge_faces).

    vertex_merge_map (N_original,): for each original vertex, the index of the nearest merged vertex (cKDTree); as in the
    reference every distance must be below 1e-6.  pre_merge_faces: a copy of the original (F_original, 3) faces."""
    verts, faces = _arrays(mesh)
    pre_merge_verts = verts.copy()
    pre_merge_faces = np.array(mesh.faces, copy=True)
    verts, faces = clean_topology(verts, faces)
    mesh.vertices = verts
    mesh.faces = faces
    distances, vertex_merge_map = cKDTree(verts).query(pre_merge_verts)
    assert np.all(distances < 1e-6), (
        "Some pre-merge vertices have no close match in the merged mesh "
        f"(max dist={distances.max():.2e}): unreferenced vertices that do not coincide with a kept one?")
    return vertex_merge_map, pre_merge_faces


@dataclass
class NormalizationParams:
    """Parameters that describe the normalization applied to a mesh (mesh_processor.py:169-174)."""
    bbox_center: Optional[np.ndarray]
    scale: float


def normalize_mesh(mesh, center: bool = True):
    """Centre the bounding box at the origin (if `center`) and scale by 2 / (largest extent), in place -> (mesh, params)."""
    verts = np.asarray(mesh.vertices, dtype=np.float64)
    bbox_center = None
    if center:
        bbox_center = (verts.min(axis=0) + verts.max(axis=0)) / 2.0
        verts = verts - bbox_center
    scale = (verts.max(axis=0) - verts.min(axis=0)).max()
    if scale > 0:
        verts = verts * (2.0 / scale)
    mesh.vertices = verts
    return mesh, NormalizationParams(bbox_center=bbox_center, scale=float(scale))


def denormalize_mesh(mesh, params: NormalizationParams):
    """Revert `normalize_mesh`, in place -> mesh."""
    verts = np.asarray(mesh.vertices, dtype=np.float64)
    if params.scale > 0:
        verts = verts * (params.scale / 2.0)
    if params.bbox_center is not None:
        verts = verts + params.bbox_center
    mesh.vertices = verts            # trimesh drops its cached face / vertex normals on assignment
    return mesh


def face_normals(verts: np.ndarray, faces: np.ndarray) -> np.ndarray:
    """Unit normals cross(v1 - v0, v2 - v0) / |.| of every face (zero for zero-area faces, as trimesh)."""
    v0, v1, v2 = (verts[faces[:, i]] for i in range(3))
    n = np.cross(v1 - v0, v2 - v0)
    norm = np.linalg.norm(n, axis=1, keepdims=True)
    return np.divide(n, norm, out=np.zeros_like(n), where=norm > 0)


def sample_surface_points(verts: np.ndarray, faces: np.ndarray, count: int, seed: int = 0) -> tuple[np.ndarray, np.ndarray]:
    """trimesh.sample.sample_surface's algorithm in float64 with `np.random.default_rng(seed).random`:
      face = searchsorted(cumsum(face areas), u * total area)            (u: `count` uniforms)
      (a, b) = two more uniforms per point (count x 2, row-major); if a + b > 1 both become |x - 1|
      point = v0 + a (v1 - v0) + b (v2 - v0)
    -> (points (count, 3) float64, face indices (count,))."""
    rand = np.random.default_rng(seed).random
    v0 = verts[faces[:, 0]]
    vecs = verts[faces[:, 1:]] - v0[:, None, :]                    # (F, 2, 3)
    area = 0.5 * np.linalg.norm(np.cross(vecs[:, 0], vecs[:, 1]), axis=1)
    cum = np.cumsum(area)
    face_index = np.searchsorted(cum, rand(count) * cum[-1])
    lengths = rand((count, 2, 1))
    fold = lengths.sum(axis=1).reshape(-1) > 1.0
    lengths[fold] -= 1.0
    lengths = np.abs(lengths)
    points = (vecs[face_index] * lengths).sum(axis=1) + v0[face_index]
    return points, face_index


def sample_surface(mesh, n_points: int, seed: int = 0, with_normals: bool = True, device=None, dtype=None) -> torch.Tensor:
    """`n_points` area-uniform samples of the surface (`sample_surface_points`), each with the unit normal of its face when
    `with_normals` -> (1, n_points, 6 | 3) tensor (float64 unless `dtype`), on `device` if given."""
    verts, faces = _arrays(mesh)
    points, face_index = sample_surface_points(verts, faces, n_points, seed)
    surface = torch.from_numpy(points)
    if with_normals:
        surface = torch.cat([surface, torch.from_numpy(face_normals(verts, faces)[face_index])], dim=-1)
    surface = surface.unsqueeze(0)
    if dtype is not None:
        surface = surface.to(dtype)
    if device is not None:
        surface = surface.to(device)
    return surface
