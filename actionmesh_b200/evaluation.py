"""ActionBench metrics on the GPU — SURVEY 8(f) rank 4 (reference actionbench/{chamfer,icp,benchmark,sample_mesh,
sample_point_cloud}.py).

Same functions, arguments, subsampling (numpy RandomState(seed) / (seed + 1) permutations) and return values as
`compute_chamfer_score` (chamfer.py:12-53) and `compute_motion_chamfer_score` (:56-89); the KD-tree nearest-neighbour queries
run as a brute-force CUDA search (amb_nearest_neighbors).  Distances are fp32 and equal an exact fp32 restatement bit for
bit, ties to the lowest index (tests/test_icp_exact_gpu.py); against the KD-tree's fp64 the scores agree to <= 1e-5
relative (tests/test_evaluation_gpu.py).

`gradient_icp` / `gradient_icp_frames` restate icp.py:53-112 on two kernels per Adam step (csrc/icp.cu, DESIGN §12): the
Chamfer loss and its gradient sums, then the closed-form backward, Adam and best-candidate tracking.  The host enqueues the
n_iter steps without waiting and reads the result back once.  `compute_chamfer_3d_4d` is benchmark.py:67-153 on top."""
from __future__ import annotations

import functools
from dataclasses import dataclass

import numpy as np
import torch

from . import ops
from ._lib import AmbError
from .mesh_input import sample_surface_points


def _cuda_points(x, device) -> torch.Tensor:
    t = torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x)
    return t.to(device=device, dtype=torch.float32).contiguous()


def compute_chamfer_score(pred, gt, n: int = 10_000, seed: int = 44, device="cuda") -> float:
    """Symmetric Chamfer distance between two point clouds (chamfer.py:12-53)."""
    dev = torch.device(device)
    if dev.type != "cuda":
        raise AmbError("actionmesh_b200.evaluation runs on CUDA only")
    rng_pred = np.random.RandomState(seed=seed)
    rng_gt = np.random.RandomState(seed=seed + 1)
    idx_pred = rng_pred.permutation(len(pred))[:n] if 0 < n < len(pred) else np.arange(len(pred))
    idx_gt = rng_gt.permutation(len(gt))[:n] if 0 < n < len(gt) else np.arange(len(gt))
    with torch.cuda.device(dev):
        p, g = _cuda_points(pred, dev), _cuda_points(gt, dev)
        d1, _ = ops.nearest_neighbors(g[torch.from_numpy(idx_gt).to(dev)], p, want_index=False)     # gt -> pred
        d2, _ = ops.nearest_neighbors(p[torch.from_numpy(idx_pred).to(dev)], g, want_index=False)   # pred -> gt
        return float(d1.double().mean() + d2.double().mean())


def compute_motion_chamfer_score(preds, gts, device="cuda") -> float:
    """Motion Chamfer distance over a sequence: correspondences from frame 0, distances over all frames (chamfer.py:56-89)."""
    dev = torch.device(device)
    if dev.type != "cuda":
        raise AmbError("actionmesh_b200.evaluation runs on CUDA only")
    with torch.cuda.device(dev):
        p, g = _cuda_points(preds, dev), _cuda_points(gts, dev)
        assert p.shape[0] == g.shape[0], "Mismatching number of timesteps"
        _, i_gt_to_pred = ops.nearest_neighbors(g[0], p[0])
        _, i_pred_to_gt = ops.nearest_neighbors(p[0], g[0])
        d1 = (p[:, i_gt_to_pred.long()] - g).double().norm(dim=-1).mean(dim=0)
        d2 = (g[:, i_pred_to_gt.long()] - p).double().norm(dim=-1).mean(dim=0)
        return float(d1.mean() + d2.mean())


# ---- gradient ICP (actionbench/icp.py) ---------------------------------------------------------------------------------


@functools.lru_cache(maxsize=1)
def _canonical_rotation_matrices() -> torch.Tensor:
    deg_to_rad = torch.pi / 180
    azim = torch.tensor([0] * 4 + [90] * 4 + [180] * 4 + [270] * 4 + [0] * 4 + [90] * 4, dtype=torch.float32) * deg_to_rad
    elev = torch.tensor([0] * 16 + [90] * 2 + [-90] * 2 + [90] * 2 + [-90] * 2, dtype=torch.float32) * deg_to_rad
    roll = torch.tensor([0, 90, 180, 270] * 4 + [0, 90] * 4, dtype=torch.float32) * deg_to_rad

    def axis(name: str, a: torch.Tensor) -> torch.Tensor:   # pytorch3d _axis_angle_rotation
        c, s, one, zero = torch.cos(a), torch.sin(a), torch.ones_like(a), torch.zeros_like(a)
        flat = {"X": (one, zero, zero, zero, c, -s, zero, s, c),
                "Y": (c, zero, s, zero, one, zero, -s, zero, c),
                "Z": (c, -s, zero, s, c, zero, zero, zero, one)}[name]
        return torch.stack(flat, -1).reshape(a.shape + (3, 3))

    return (axis("X", azim) @ axis("Y", elev)) @ axis("Z", roll)


def canonical_rotation_matrices() -> torch.Tensor:
    """The 24 initial rotations of icp.py:18-50, (24, 3, 3) fp32 on the CPU: pytorch3d's euler_angles_to_matrix(..., "XYZ")
    of the fp32 angles, evaluated the way pytorch3d does (cos, sin, X @ Y @ Z in fp32).  cos(pi/2) is not 0 in fp32, so the
    matrices carry off-diagonal residues of ~8.7e-8; they are part of the reference and are kept.  These are constants of
    the algorithm, computed once on the host."""
    return _canonical_rotation_matrices().clone()


@dataclass
class IcpTransform:
    """Per-frame result of `gradient_icp_frames`: packed (F, 16) fp32 = best loss, R (9, row-major), T (3), s (3)."""
    packed: torch.Tensor

    @property
    def loss(self) -> torch.Tensor:
        return self.packed[:, 0]

    @property
    def R(self) -> torch.Tensor:
        return self.packed[:, 1:10].reshape(-1, 3, 3)

    @property
    def T(self) -> torch.Tensor:
        return self.packed[:, 10:13]

    @property
    def s(self) -> torch.Tensor:
        return self.packed[:, 13:16]

    def __len__(self) -> int:
        return self.packed.shape[0]

    def __getitem__(self, k: int) -> "IcpTransform":
        return IcpTransform(self.packed[k:k + 1])

    def transform_points(self, points: torch.Tensor) -> torch.Tensor:
        """(p * s) @ R + T on the GPU, frame f of (F, N, 3) points by transform f; a single transform applies to every
        frame, and (N, 3) points are one frame."""
        one = points.dim() == 2
        p = points[None] if one else points
        with torch.cuda.device(self.packed.device):
            out = ops.icp_transform_points(p.to(self.packed.device, torch.float32), self.packed[:, 1:])
        return out[0] if one else out


def gradient_icp_frames(pc_pred: torch.Tensor, pc_gt: torch.Tensor, lr: float = 0.01, n_iter: int = 200) -> IcpTransform:
    """`gradient_icp` of every frame at once: pred (F, P, 3) and gt (F, Q, 3) fp32 CUDA tensors -> IcpTransform (F)."""
    if pc_pred.dim() != 3 or pc_gt.dim() != 3 or pc_pred.shape[0] != pc_gt.shape[0]:
        raise AmbError(f"gradient_icp_frames: expected (F, P, 3) and (F, Q, 3) points, got {tuple(pc_pred.shape)} and "
                       f"{tuple(pc_gt.shape)}")
    if not pc_pred.is_cuda:
        raise AmbError("gradient_icp_frames: expected CUDA tensors (there is no CPU fallback)")
    dev = pc_pred.device
    with torch.cuda.device(dev):
        pred, gt = pc_pred.contiguous(), pc_gt.contiguous()
        F = pred.shape[0]
        rot_init = canonical_rotation_matrices().to(dev)
        nc = rot_init.shape[0]
        # the reference's initial state: T = 0, d6 = (1, 0, 0, 0, 1, 0), s = 1, so R = R_init exactly
        params = torch.zeros(F, nc, 12, dtype=torch.float32, device=dev)
        params[..., 3] = 1.0
        params[..., 7] = 1.0
        params[..., 9:] = 1.0
        rot = rot_init.repeat(F, 1, 1, 1)            # a copy: the Adam step rewrites it every step
        adam_m, adam_v = torch.zeros_like(params), torch.zeros_like(params)
        best = torch.zeros(F, 16, dtype=torch.float32, device=dev)
        best[:, 0] = float("inf")
        sums = torch.empty(F, nc, 13, dtype=torch.float64, device=dev)
        scratch = torch.empty(ops.icp_scratch_doubles(F, nc, pred.shape[1], gt.shape[1]), dtype=torch.float64, device=dev)
        for it in range(n_iter):
            ops.icp_chamfer_grad(pred, gt, rot, params, out=sums, scratch=scratch)
            ops.icp_adam_step(sums, rot_init, it + 1, lr, params, adam_m, adam_v, rot, best)
        if not bool(torch.isfinite(best[:, 0]).all()):   # the one read-back
            raise AmbError("gradient_icp: no candidate reached a finite loss (the reference fails here too)")
    return IcpTransform(best)


def gradient_icp(pc_pred: torch.Tensor, pc_gt: torch.Tensor, lr: float = 0.01, n_iter: int = 200) -> IcpTransform:
    """Rigid + anisotropic-scale alignment of pred (P, 3) to gt (Q, 3) (icp.py:53-112) -> IcpTransform of one frame:
    transform_points(p) = (p * s) @ R + T."""
    return gradient_icp_frames(pc_pred[None], pc_gt[None], lr=lr, n_iter=n_iter)


# ---- point sampling (actionbench/sample_point_cloud.py, sample_mesh.py) ------------------------------------------------


def sample_point_cloud(point_cloud: torch.Tensor, n_pts: int, seed: int = 44) -> torch.Tensor:
    """(T, N, C) -> (T, n_pts, C): one seeded RandomState permutation shared by every frame (sample_point_cloud.py:11-36)."""
    n_src = point_cloud.shape[1]
    if n_src <= n_pts:
        return point_cloud
    idx = torch.from_numpy(np.random.RandomState(seed=seed).permutation(n_src)[:n_pts]).long()
    return point_cloud[:, idx.to(point_cloud.device)]


def _mesh_arrays(mesh) -> tuple[np.ndarray, np.ndarray]:
    return np.asarray(mesh.vertices), np.asarray(mesh.faces, dtype=np.int64).reshape(-1, 3)


def _synchronized_sampling(verts: np.ndarray, faces: np.ndarray, n_pts: int, seed: int):
    """pytorch3d's draws in get_baryc_sampling_mesh (sample_mesh.py:58-103) on a CPU generator seeded with `seed`: face
    indices from multinomial(fp32 face areas, n, replacement=True), then u, v = rand(2, 1, n) -> barycentric weights."""
    v = verts.astype(np.float32)
    v0, v1, v2 = (v[faces[:, i]] for i in range(3))
    a, b = v1 - v0, v2 - v0                                   # pytorch3d mesh_face_areas_normals, fp32
    cx = a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1]
    cy = a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2]
    cz = a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]
    areas = np.sqrt(cx * cx + cy * cy + cz * cz) / np.float32(2.0)
    gen = torch.Generator().manual_seed(seed)
    face_idx = torch.from_numpy(areas[None]).multinomial(n_pts, replacement=True, generator=gen)[0].numpy()
    uv = torch.rand(2, 1, n_pts, dtype=torch.float32, generator=gen).numpy()
    u_sqrt = np.sqrt(uv[0, 0])
    w = (np.float32(1.0) - u_sqrt, u_sqrt * (np.float32(1.0) - uv[1, 0]), u_sqrt * uv[1, 0])
    return face_idx, w


def sample_meshes(meshes: list, n_pts: int = 100_000, synchronized: bool = False, seed: int = 44) -> torch.Tensor:
    """(T, n_pts, 3) fp32 CPU samples of T meshes (objects with .vertices and .faces), as sample_mesh.py:211-243.

    Unsynchronized: mesh i is sampled area-uniformly with seed + i (trimesh's sample_surface, restated by
    mesh_input.sample_surface_points).  Synchronized: face indices and barycentric weights are drawn once on mesh 0 (see
    `_synchronized_sampling`) and applied to every frame, which must share mesh 0's faces."""
    if not synchronized:
        return torch.stack([torch.from_numpy(sample_surface_points(*_mesh_arrays(m), n_pts, seed + i)[0]).float()
                            for i, m in enumerate(meshes)])
    arrays = [_mesh_arrays(m) for m in meshes]
    faces = arrays[0][1]
    assert all(np.array_equal(faces, f) for _, f in arrays), "synchronized sampling needs one face array for every frame"
    face_idx, (w0, w1, w2) = _synchronized_sampling(arrays[0][0], faces, n_pts, seed)
    out = np.empty((len(arrays), n_pts, 3), dtype=np.float32)
    for k, (verts, _) in enumerate(arrays):
        v = verts.astype(np.float32)
        a, b, c = (v[faces[face_idx, i]] for i in range(3))
        out[k] = w0[:, None] * a + w1[:, None] * b + w2[:, None] * c
    return torch.from_numpy(out)


# ---- CD-3D / CD-4D / CD-M (actionbench/benchmark.py) ----------------------------------------------------------------------


def compute_chamfer_3d_4d(gt_pc, pred_meshes: list, device="cuda", is_4D: bool = False, n_pts_icp: int = 10_000,
                          n_pts_chamfer: int = 100_000, seed: int = 44) -> tuple[float, float, float]:
    """(cd_3d, cd_4d, cd_motion) of T predicted meshes against gt points (T, N, 3), as benchmark.py:67-153.

    cd_3d aligns each frame by its own ICP, cd_4d every frame by frame 0's ICP, and cd_motion (is_4D only) scores
    synchronized samples under frame 0's ICP with the motion Chamfer distance.  The reference runs frame 0's ICP twice (per
    frame and "unified") on identical inputs; the kernels are deterministic, so the two runs would give identical bits, and
    the per-frame result is reused."""
    dev = torch.device(device)
    if dev.type != "cuda":
        raise AmbError("actionmesh_b200.evaluation runs on CUDA only")
    gt = torch.as_tensor(np.asarray(gt_pc) if not torch.is_tensor(gt_pc) else gt_pc).float()
    if gt.shape[0] != len(pred_meshes):
        raise AmbError(f"compute_chamfer_3d_4d: {gt.shape[0]} gt frames for {len(pred_meshes)} meshes")
    pred_pc = sample_meshes(pred_meshes, n_pts=n_pts_chamfer, synchronized=False, seed=seed)
    pred_icp = sample_point_cloud(pred_pc, n_pts=n_pts_icp, seed=seed)
    gt_icp = sample_point_cloud(gt, n_pts=n_pts_icp, seed=seed)
    with torch.cuda.device(dev):
        pred_pc, gt_d = pred_pc.to(dev), gt.to(dev)
        per_frame = gradient_icp_frames(pred_icp.to(dev), gt_icp.to(dev))
        unified = per_frame[0]
        aligned_3d = per_frame.transform_points(pred_pc)
        aligned_u4d = unified.transform_points(pred_pc)
        n_ts = len(pred_meshes)
        cd_3d = np.mean([compute_chamfer_score(gt=gt_d[k], pred=aligned_3d[k], device=dev) for k in range(n_ts)])
        cd_4d = np.mean([compute_chamfer_score(gt=gt_d[k], pred=aligned_u4d[k], device=dev) for k in range(n_ts)])
        cd_motion = 0.0
        if is_4D:
            pred_4d = sample_meshes(pred_meshes, n_pts=n_pts_chamfer, synchronized=True, seed=seed).to(dev)
            cd_motion = compute_motion_chamfer_score(preds=unified.transform_points(pred_4d), gts=gt_d, device=dev)
    return float(cd_3d), float(cd_4d), float(cd_motion)
