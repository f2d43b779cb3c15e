"""B200MeshPostprocessor: the reference's MeshPostprocessor (actionmesh/preprocessing/mesh_processor.py:374-425) with the
decimation and floater removal on the GPU (csrc/mesh_process.cu).

`process_mesh(mesh)` runs the reference's steps in the reference's order:
  1. clean on the host: `mesh_input.clean_topology` (merge at 8 decimals, drop degenerate faces, drop duplicate faces, drop
     unreferenced vertices), the rules of trimesh's merge_vertices / remove_degenerate_faces / remove_duplicate_faces /
     remove_unreferenced_vertices;
  2. decimate to `face_decimation` faces (only when it is not -1 and the mesh has more faces): parallel greedy quadric edge
     collapse in rounds, in place of trimesh's simplify_quadric_decimation (fast_simplification);
  3. remove floaters (only when `floaters_threshold` > 0): drop the components with fewer than
     int(largest component's faces * threshold) faces, components being faces joined through edges held by exactly two faces,
     as trimesh's split(only_watertight=False).
DESIGN.md §15 gives the algorithm and its invariants.  Differences from the reference:
  - the input mesh is not modified (the reference cleans its input in place; nothing downstream reads the input afterwards);
  - the decimation is a different algorithm from fast_simplification's, so the vertices differ; it is deterministic, which is
    why `seed` is accepted and unused;
  - floater removal keeps the kept faces and their vertices in their original order, where trimesh concatenates the kept
    components one after another and duplicates a vertex shared by two kept components that touch only there.  The geometry
    is the same.
"""
from __future__ import annotations

import logging
from typing import Optional

import numpy as np
import torch

from . import ops
from .mesh_input import clean_topology

logger = logging.getLogger(__name__)


def _round_limit(winners: np.ndarray, n_faces: int, target: int) -> tuple[int, int]:
    """(key limit, faces removed) of the round whose winners would pass `target`: only the cheapest winners, in key order, up
    to the first that reaches it.  winners: (n, 2) int64 (key bits, face count)."""
    keys = winners[:, 0].view(np.uint64)
    order = np.argsort(keys, kind="stable")
    cum = np.cumsum(winners[order, 1])
    k = int(np.argmax(n_faces - cum <= target))
    return int(keys[order[k]]), int(cum[k])


def decimate(positions: torch.Tensor, faces: torch.Tensor, target: int, work: torch.Tensor,
             scan: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor, int]:
    """Quadric edge-collapse decimation of a clean mesh on its device down to `target` faces (closed meshes end at target - 1
    or target; stops above it when no valid collapse is left) -> (positions (V', 3) fp64, faces (F', 3) int32, rounds).
    `positions` is updated in place."""
    V, F = positions.shape[0], faces.shape[0]
    quadrics = None
    rounds = 0
    while F > target:
        adj = ops.mesh_adjacency(faces, V, work, scan)
        if quadrics is None:
            quadrics = ops.mesh_quadrics(positions, faces, adj)
        sel = ops.mesh_collapse_select(positions, quadrics, faces, adj)
        if not len(sel["winners"]):
            logger.warning(f"[Decimation] No valid edge collapse left at {F:,} faces (target {target:,})")
            break
        limit, removed = ops.NO_KEY, sel["removed"]
        if F - removed < target:
            limit, removed = _round_limit(sel["winners"].cpu().numpy(), F, target)
        remap = ops.mesh_collapse_apply(adj[3], sel, limit, positions, quadrics)
        faces = ops.mesh_compact_faces(faces, scan, remap=remap)
        assert faces.shape[0] == F - removed
        F = faces.shape[0]
        rounds += 1
    positions, faces = ops.mesh_compact_vertices(positions, faces, work, scan)
    return positions, faces, rounds


def remove_floaters(positions: torch.Tensor, faces: torch.Tensor, threshold: float, work: torch.Tensor,
                    scan: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """The reference's remove_floaters rule (mesh_processor.py:288-325) on the device; returns the inputs unchanged when the
    mesh has <= 1 component or no component is kept."""
    F = faces.shape[0]
    adj = ops.mesh_adjacency(faces, positions.shape[0], work, scan)
    labels, sizes = ops.mesh_face_components(adj[3], F)
    counts = sizes.cpu().numpy()
    n_components = int(np.count_nonzero(counts))
    if n_components <= 1:
        logger.debug(f"[Floaters] Skipped: mesh has {n_components} component(s)")
        return positions, faces
    min_faces = int(int(counts.max()) * threshold)
    kept = int(np.count_nonzero(counts[counts > 0] >= min_faces))
    if not kept:
        logger.warning(f"[Floaters] No components kept after filtering (threshold={threshold}, min_faces={min_faces}), "
                       "returning original mesh")
        return positions, faces
    logger.info(f"[Floaters] Removed {n_components - kept} component(s): {n_components} -> {kept}")
    faces = ops.mesh_compact_faces(faces, scan, labels=labels, sizes=sizes, min_size=min_faces)
    return ops.mesh_compact_vertices(positions, faces, work, scan)


def make_mesh(vertices: np.ndarray, faces: np.ndarray):
    """trimesh.Trimesh(v, f, process=False) when trimesh is installed, else the package's AnchorMesh with vertex normals."""
    try:
        import trimesh

        return trimesh.Trimesh(vertices=vertices, faces=faces, process=False)
    except ImportError:
        from .pipeline import _vertex_normals
        from .triposg_vae import AnchorMesh

        vt = torch.from_numpy(vertices)
        n = _vertex_normals(vt, torch.from_numpy(faces)) if len(faces) else torch.zeros_like(vt)
        return AnchorMesh(vertices=vertices, faces=faces, vertex_normals=n.numpy())


class B200MeshPostprocessor:
    """Drop-in for the reference's `MeshPostprocessor` (same constructor and `process_mesh(mesh, seed)`), with decimation and
    floater removal on `device`.  Select it with `config_updates={"model.mesh_process._target_":
    "actionmesh_b200.mesh_process.B200MeshPostprocessor"}` or by assigning `pipe.mesh_process`."""

    def __init__(self, bounds=(-1.005, -1.005, -1.005, 1.005, 1.005, 1.005), face_decimation: int = -1,
                 floaters_threshold: float = 0.0, verbose: bool = True, *, device="cuda"):
        assert bounds[0] == bounds[1] == bounds[2]
        assert bounds[3] == bounds[4] == bounds[5]
        self.bounds = tuple(bounds)
        self.face_decimation = face_decimation
        self.floaters_threshold = floaters_threshold
        self.verbose = verbose
        self.device = torch.device(device)

    @torch.no_grad()
    def process_mesh(self, mesh, seed: Optional[int] = None):
        """Clean, decimate and remove floaters -> a new mesh with .vertices (float64), .faces and .vertex_normals; `mesh` (any
        object with .vertices / .faces) is not modified.  `seed` is unused: every step is deterministic."""
        verts, faces = clean_topology(np.asarray(mesh.vertices, dtype=np.float64),
                                      np.asarray(mesh.faces, dtype=np.int64).reshape(-1, 3))
        if not np.isfinite(verts).all():
            raise ValueError("process_mesh: the mesh has non-finite vertices")
        decimating = self.face_decimation != -1 and len(faces) > self.face_decimation
        if self.face_decimation != -1 and not decimating and self.verbose:
            logger.info(f"[Decimation] Skipped: mesh has {len(faces):,} faces (<= target {self.face_decimation:,})")
        if (decimating or self.floaters_threshold > 0.0) and len(faces):
            if self.device.type != "cuda":
                raise ops._lib.AmbError("B200MeshPostprocessor runs on CUDA (sm_90a) only; there is no CPU fallback")
            with torch.cuda.device(self.device):
                pos = torch.from_numpy(verts).to(self.device)
                f = torch.from_numpy(faces.astype(np.int32)).to(self.device)
                work, scan = ops.mesh_scan_scratch(len(verts), len(faces), self.device)
                if decimating:
                    if self.verbose:
                        logger.info(f"[Decimation] Before: {len(faces):,} faces")
                    pos, f, _ = decimate(pos, f, int(self.face_decimation), work, scan)
                    if self.verbose:
                        logger.info(f"[Decimation] After: {f.shape[0]:,} faces")
                if self.floaters_threshold > 0.0:
                    pos, f = remove_floaters(pos, f, float(self.floaters_threshold), work, scan)
                verts, faces = pos.cpu().numpy(), f.cpu().numpy().astype(np.int64)
        return make_mesh(verts, faces)
