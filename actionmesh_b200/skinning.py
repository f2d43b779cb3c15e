"""Bones and skin weights fitted to a fixed-topology vertex animation, on the GPU: the data a skinned GLB holds.

    fit = fit_skinning(vertices (T, V, 3), n_bones)      -> SkinningFit
    gltf.write_skinned_glb(path, fit, faces)

The model is Smooth Skinning Decomposition with Rigid Bones (SSDR, Le & Deng 2012): v^_i^t = sum_j w_ij (R_j^t p_i + t_j^t)
with w_ij >= 0, sum_j w_ij = 1 and at most 4 non-zero weights per vertex, p_i being the rest pose vertices[0].  It is fitted
by alternating least squares in the fp64 kernels of csrc/skinning.cu (every rule is in DESIGN.md §20):

  1. seeds: farthest-point sampling of n_bones rest vertices; every vertex starts on its nearest seed's bone.
  2. CLUSTER_ROUNDS rounds of rigid clustering: each bone's transforms fitted to its vertices (one-hot weights), then every
     vertex moved to its lowest-error bone; a bone left without vertices takes the worst-fit vertex.
  3. `iterations` rounds of: every bone's transforms refitted in bone order, then every vertex's weights.
Neither step of a round can increase the error (DESIGN.md §20 says why), so `history` does not increase.
"""
from __future__ import annotations

import logging
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from . import ops

logger = logging.getLogger(__name__)

MAX_BONES = 256        # JOINTS_0 is written as u8
CLUSTER_ROUNDS = 5
DEFAULT_ITERATIONS = 20


@dataclass
class SkinningFit:
    """A skinned animation: rest (V, 3) fp64; joints (V, 4) int32 and weights (V, 4) fp64 (unused slots: joint 0, weight 0);
    rotations (T, B, 3, 3) and translations (T, B, 3) fp64, bone j mapping a rest point p to R p + t in frame t; centres
    (B, 3) fp64, each bone's weighted rest centre (where its joint is placed); history: sum_t,i |v^ - v|^2 after the
    initialisation and after every iteration; rms_error and max_error: the final RMS and largest |v^ - v| over vertices and
    frames, relative to the diagonal of the rest pose's bounding box."""
    rest: np.ndarray
    joints: np.ndarray
    weights: np.ndarray
    rotations: np.ndarray
    translations: np.ndarray
    centres: np.ndarray
    history: list
    rms_error: float
    max_error: float

    @property
    def n_bones(self) -> int:
        return self.rotations.shape[1]


def _check(vertices: np.ndarray, n_bones: int) -> None:
    if vertices.ndim != 3 or vertices.shape[2] != 3 or vertices.shape[0] < 1 or vertices.shape[1] < 1:
        raise ValueError(f"vertices must be (T, V, 3) with T >= 1 and V >= 1, got {vertices.shape}")
    if not np.isfinite(vertices).all():
        raise ValueError("vertices contain a non-finite value")
    n_max = min(vertices.shape[1], MAX_BONES)
    if not 1 <= n_bones <= n_max:
        raise ValueError(f"n_bones must be in [1, {n_max}] for {vertices.shape[1]} vertices, got {n_bones}")


def _reseed(labels: np.ndarray, min_error: np.ndarray, n_bones: int) -> np.ndarray:
    """Every bone without a vertex, in bone order, takes the next worst-fit vertex (largest error, ties to the lowest index)."""
    empty = np.flatnonzero(np.bincount(labels, minlength=n_bones) == 0)
    if len(empty):
        worst = np.argsort(-min_error, kind="stable")[:len(empty)]
        labels = labels.copy()
        labels[worst] = empty
    return labels


def fit_skinning(vertices, n_bones: int, iterations: int = DEFAULT_ITERATIONS,
                 device: Optional[torch.device] = None) -> SkinningFit:
    """Fit `n_bones` rigid bones and <= 4 skin weights per vertex to the (T, V, 3) animation `vertices` (rest pose
    vertices[0]) -> SkinningFit.  ValueError: a non-finite value, T < 1, or n_bones outside [1, min(V, 256)]."""
    v = np.ascontiguousarray(vertices, dtype=np.float64)
    _check(v, int(n_bones))
    if iterations < 0:
        raise ValueError(f"iterations must be >= 0, got {iterations}")
    B = int(n_bones)
    T, V, _ = v.shape
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(dev):
        verts = torch.from_numpy(v).to(dev)
        rest = verts[0].contiguous()
        eye = np.zeros((T, B, 12))
        eye[:, :, [0, 4, 8]] = 1.0
        xf = torch.from_numpy(eye).to(dev)
        scratch = ops.skin_scratch(T, V, dev)
        _, labels, centres = ops.skin_seeds(rest, B)
        joints = torch.zeros(V, 4, dtype=torch.int32, device=dev)
        weights = torch.zeros(V, 4, dtype=torch.float64, device=dev)
        weights[:, 0] = 1.0

        def refit_bones():
            for j in range(B):
                ops.skin_bone_update(rest, verts, xf, joints, weights, j, centres, scratch)

        for _ in range(CLUSTER_ROUNDS):
            joints[:, 0] = labels
            refit_bones()
            argmin, min_error, _ = ops.skin_rigid_error(rest, verts, xf)
            labels = torch.from_numpy(_reseed(argmin.cpu().numpy(), min_error.cpu().numpy(), B)).to(dev)
        joints[:, 0] = labels
        history = [float(ops.skin_error(rest, verts, xf, joints, weights, scratch)[0][T])]
        for _ in range(iterations):
            refit_bones()
            _, _, cand = ops.skin_rigid_error(rest, verts, xf)
            ops.skin_weight_update(rest, verts, xf, cand, joints, weights)
            history.append(float(ops.skin_error(rest, verts, xf, joints, weights, scratch)[0][T]))
        frame_errors, max_error2 = ops.skin_error(rest, verts, xf, joints, weights, scratch)
        transforms = xf.cpu().numpy()
        fit_joints, fit_weights, fit_centres = joints.cpu().numpy(), weights.cpu().numpy(), centres.cpu().numpy()
        total, max2 = float(frame_errors[T]), float(max_error2[0])
    diag = float(np.linalg.norm(v[0].max(0) - v[0].min(0)))
    scale = 1.0 / diag if diag > 0 else 1.0
    fit = SkinningFit(rest=v[0].copy(), joints=fit_joints, weights=fit_weights,
                      rotations=transforms[:, :, :9].reshape(T, B, 3, 3).copy(), translations=transforms[:, :, 9:].copy(),
                      centres=fit_centres, history=history, rms_error=float(np.sqrt(total / (T * V))) * scale,
                      max_error=float(np.sqrt(max2)) * scale)
    logger.info(f"Skinning fit: {B} bones, {T} frames x {V} vertices, RMS error {fit.rms_error:.3e} and max error "
                f"{fit.max_error:.3e} of the rest bounding-box diagonal")
    return fit
