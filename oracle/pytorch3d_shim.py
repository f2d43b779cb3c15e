"""TEST INFRASTRUCTURE ONLY.  Minimal in-memory stand-in for the pytorch3d pieces ActionBench imports.

pytorch3d is an unpinned third-party dependency of the reference's benchmark (actionbench/icp.py, sample_mesh.py), neither
vendored under the reference checkout nor installed here.  What follows restates its documented semantics, with autograd, for
exactly the calls the benchmark makes:
    icp.py:8-13            chamfer_distance (brute force), euler_angles_to_matrix, rotation_6d_to_matrix,
                           transform3d.{Transform3d, Scale, Rotate, Translate} with compose / stack / transform_points
    sample_mesh.py:9-11    ops.mesh_face_areas_normals, ops.packed_to_padded, structures.{Meshes, join_meshes_as_batch}
"pytorch3d semantics unpinned": there is no wheel here to check this file against.
"""
from __future__ import annotations

import functools
import sys
import types

import torch
import torch.nn.functional as F


# ---- pytorch3d.loss ------------------------------------------------------------------------------------------------------

def chamfer_distance(x, y, batch_reduction="mean", point_reduction="mean", norm=2, single_directional=False):
    """Squared-L2 Chamfer distance of (N, P, 3) and (N, Q, 3) batches -> (loss, None): mean over points of each
    direction's nearest squared distance, summed over both directions, batch-reduced by "mean", "sum" or None."""
    assert norm == 2 and point_reduction == "mean" and not single_directional
    d = torch.cdist(x, y) ** 2 if x.shape[1] * y.shape[1] > 1 << 22 else ((x[:, :, None] - y[:, None]) ** 2).sum(-1)
    loss = d.min(2).values.mean(1) + d.min(1).values.mean(1)
    if batch_reduction == "mean":
        loss = loss.mean()
    elif batch_reduction == "sum":
        loss = loss.sum()
    return loss, None


# ---- pytorch3d.transforms ------------------------------------------------------------------------------------------------

def _axis_angle_rotation(axis: str, angle: torch.Tensor) -> torch.Tensor:
    cos, sin = torch.cos(angle), torch.sin(angle)
    one, zero = torch.ones_like(angle), torch.zeros_like(angle)
    if axis == "X":
        flat = (one, zero, zero, zero, cos, -sin, zero, sin, cos)
    elif axis == "Y":
        flat = (cos, zero, sin, zero, one, zero, -sin, zero, cos)
    else:
        flat = (cos, -sin, zero, sin, cos, zero, zero, zero, one)
    return torch.stack(flat, -1).reshape(angle.shape + (3, 3))


def euler_angles_to_matrix(euler_angles: torch.Tensor, convention: str) -> torch.Tensor:
    mats = [_axis_angle_rotation(c, e) for c, e in zip(convention, torch.unbind(euler_angles, -1))]
    return functools.reduce(torch.matmul, mats)


def rotation_6d_to_matrix(d6: torch.Tensor) -> torch.Tensor:
    """Gram-Schmidt of the two 3-vectors (Zhou et al. 2019): rows b1, b2, b1 x b2."""
    a1, a2 = d6[..., :3], d6[..., 3:]
    b1 = F.normalize(a1, dim=-1)
    b2 = a2 - (b1 * a2).sum(-1, keepdim=True) * b1
    b2 = F.normalize(b2, dim=-1)
    b3 = torch.cross(b1, b2, dim=-1)
    return torch.stack((b1, b2, b3), dim=-2)


class Transform3d:
    """Row-vector homogeneous transforms: points @ M; compose(a, b) applies self, then a, then b."""

    def __init__(self, matrix: torch.Tensor | None = None, dtype=torch.float32, device="cpu"):
        self._matrix = torch.eye(4, dtype=dtype, device=device)[None] if matrix is None else matrix
        self._transforms = []

    def get_matrix(self) -> torch.Tensor:
        m = self._matrix
        for t in self._transforms:
            m = m @ t.get_matrix()
        return m

    def compose(self, *others) -> "Transform3d":
        out = Transform3d(self._matrix.clone())
        out._transforms = self._transforms + list(others)
        return out

    def stack(self, *others) -> "Transform3d":
        return Transform3d(torch.cat([t.get_matrix() for t in (self, *others)], dim=0))

    def transform_points(self, points: torch.Tensor, eps=None) -> torch.Tensor:
        pts = points[None] if points.dim() == 2 else points
        m = self.get_matrix()
        homog = torch.cat([pts, torch.ones_like(pts[..., :1])], dim=-1)
        out = homog @ m
        denom = out[..., 3:]
        if eps is not None:
            denom = denom.sign() * denom.abs().clamp(min=eps)
        out = out[..., :3] / denom
        return out[0] if points.dim() == 2 and out.shape[0] == 1 else out


class Scale(Transform3d):
    def __init__(self, s: torch.Tensor):
        m = torch.eye(4, dtype=s.dtype, device=s.device).repeat(s.shape[0], 1, 1)
        m[:, 0, 0], m[:, 1, 1], m[:, 2, 2] = s[:, 0], s[:, 1], s[:, 2]
        super().__init__(m)


class Rotate(Transform3d):
    def __init__(self, R: torch.Tensor):
        m = torch.eye(4, dtype=R.dtype, device=R.device).repeat(R.shape[0], 1, 1)
        m[:, :3, :3] = R
        super().__init__(m)


class Translate(Transform3d):
    def __init__(self, T: torch.Tensor):
        m = torch.eye(4, dtype=T.dtype, device=T.device).repeat(T.shape[0], 1, 1)
        m[:, 3, :3] = T
        super().__init__(m)


# ---- pytorch3d.ops -------------------------------------------------------------------------------------------------------

def mesh_face_areas_normals(verts: torch.Tensor, faces: torch.Tensor):
    """(areas (F,), unit normals (F, 3)): n = (v1 - v0) x (v2 - v0) componentwise, area = |n| / 2, normal n / max(|n|, 1e-6)."""
    v0, v1, v2 = (verts[faces[:, i]] for i in range(3))
    a, b = v1 - v0, v2 - v0
    n = torch.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                     a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], dim=1)
    norm = torch.sqrt(n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1] + n[:, 2] * n[:, 2])
    return norm / 2.0, n / norm.clamp_min(1e-6)[:, None]


def packed_to_padded(inputs: torch.Tensor, first_idxs: torch.Tensor, max_size: int) -> torch.Tensor:
    out = torch.zeros((first_idxs.shape[0], max_size) + inputs.shape[1:], dtype=inputs.dtype, device=inputs.device)
    bounds = first_idxs.tolist() + [inputs.shape[0]]
    for i in range(first_idxs.shape[0]):
        out[i, :bounds[i + 1] - bounds[i]] = inputs[bounds[i]:bounds[i + 1]]
    return out


# ---- pytorch3d.structures ------------------------------------------------------------------------------------------------

class Meshes:
    def __init__(self, verts: list, faces: list):
        self._verts, self._faces = list(verts), list(faces)
        self.device = self._verts[0].device if self._verts else torch.device("cpu")
        self.valid = torch.tensor([len(f) > 0 for f in self._faces], dtype=torch.bool)

    def __len__(self):
        return len(self._verts)

    def __getitem__(self, k):
        return Meshes([self._verts[k]], [self._faces[k]])

    def isempty(self) -> bool:
        return len(self._verts) == 0 or all(len(f) == 0 for f in self._faces)

    def verts_packed(self):
        return torch.cat(self._verts)

    def faces_packed(self):
        offs = [0]
        for v in self._verts[:-1]:
            offs.append(offs[-1] + len(v))
        return torch.cat([f + o for f, o in zip(self._faces, offs)])

    def faces_list(self):
        return self._faces

    def num_faces_per_mesh(self):
        return torch.tensor([len(f) for f in self._faces])

    def mesh_to_faces_packed_first_idx(self):
        n = self.num_faces_per_mesh()
        return torch.cumsum(n, 0) - n


def join_meshes_as_batch(meshes: list) -> Meshes:
    return Meshes([v for m in meshes for v in m._verts], [f for m in meshes for f in m._faces])


def install() -> None:
    """Register the stand-in as `pytorch3d` and its submodules in sys.modules."""
    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        m._AMB_SHIM = True
        sys.modules[name] = m
        return m

    t3d = mod("pytorch3d.transforms.transform3d", Transform3d=Transform3d, Scale=Scale, Rotate=Rotate, Translate=Translate)
    mod("pytorch3d.transforms", transform3d=t3d, euler_angles_to_matrix=euler_angles_to_matrix,
        rotation_6d_to_matrix=rotation_6d_to_matrix)
    mod("pytorch3d.loss", chamfer_distance=chamfer_distance)
    mod("pytorch3d.ops.mesh_face_areas_normals", mesh_face_areas_normals=mesh_face_areas_normals)
    mod("pytorch3d.ops.packed_to_padded", packed_to_padded=packed_to_padded)
    mod("pytorch3d.ops", mesh_face_areas_normals=mesh_face_areas_normals, packed_to_padded=packed_to_padded)
    mod("pytorch3d.structures", Meshes=Meshes, join_meshes_as_batch=join_meshes_as_batch)
    mod("pytorch3d")
