"""The joint rotations of a rigged mesh input's own skeleton fitted to the vertex animation, on the GPU.

    rig = gltf.load_rig(path)                                   -> GltfRig
    fit = fit_rig_animation(rig, vertices (T, V, 3))            -> RigFit
    gltf.write_rig_animation(path, out_path, rig, fit)

The model (DESIGN.md §21): per frame, a local rotation R_j for every joint and a local translation tau_j for root joints
only; every other local translation, every local scale and every non-joint node keep their default values.
G_j = G_parent T(tau_j) R_j S_j and v^_i = sum_s w_is G_{j_s} B_s p_i.  Every frame starts at the default pose; a sweep
visits the joints in topological order and replaces R_j, then (for a root) tau_j, by the exact minimiser of the squared
error with everything else fixed, so `history` does not increase.  The fp64 kernels are in csrc/rig.cu.
"""
from __future__ import annotations

import logging
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from . import ops

logger = logging.getLogger(__name__)

DEFAULT_SWEEPS = 200


@dataclass
class RigFit:
    """A joint animation of a `gltf.GltfRig`, joints in the skin's order: rotations (T, J, 4) unit quaternions (x, y, z, w)
    and rotation_matrices (T, J, 3, 3) fp64, the local rotation of every joint in frame t; translations (T, J, 3) fp64,
    the local translations (only root joints' differ from the default); history: sum_t,i |v^ - v|^2 after the
    initialisation and after every sweep; rms_error and max_error: the final RMS and largest |v^ - v| over vertices and
    frames, relative to the diagonal of the rest pose's bounding box."""
    rotations: np.ndarray
    rotation_matrices: np.ndarray
    translations: np.ndarray
    history: list
    rms_error: float
    max_error: float


@dataclass
class RigArrays:
    """A `GltfRig` as the kernels take it, joints renumbered in the rig's topological order `order` (depth-first, so the
    subtree of joint k is [k, subtree_end[k])): parent (J) int32; scale (J, 3); above (J, 12) and above_inv (J, 9), the
    fixed transform above each root and the inverse of its linear part (zero rows for other joints); binds (NB, 12) and
    bind_joint (NB) int32; rotations (J, 9) and translations (J, 3), the default local pose; points and rest (V, 3);
    slot_bind (V, 8) int32 and slot_weight (V, 8); lists: one int32 array, joint k's vertices being
    lists[offsets[k]:offsets[k + 1]] in ascending order."""
    order: np.ndarray
    parent: np.ndarray
    subtree_end: np.ndarray
    scale: np.ndarray
    above: np.ndarray
    above_inv: np.ndarray
    binds: np.ndarray
    bind_joint: np.ndarray
    rotations: np.ndarray
    translations: np.ndarray
    points: np.ndarray
    rest: np.ndarray
    slot_bind: np.ndarray
    slot_weight: np.ndarray
    lists: np.ndarray
    offsets: np.ndarray


@dataclass
class RigTensors:
    """`RigArrays` on the device, with the kernels' outputs and scratch for T frames (the argument of the ops.rig_*)."""
    parent: torch.Tensor
    scale: torch.Tensor
    above: torch.Tensor
    above_inv: torch.Tensor
    binds: torch.Tensor
    bind_joint: torch.Tensor
    points: torch.Tensor
    rest: torch.Tensor
    slot_bind: torch.Tensor
    slot_weight: torch.Tensor
    world: torch.Tensor
    skin: torch.Tensor
    scratch: torch.Tensor


def _xf12(m: np.ndarray) -> np.ndarray:
    """(..., 4, 4) affine matrices -> (..., 12): the 3x3 linear part row-major, then the translation."""
    m = np.asarray(m, np.float64)
    return np.concatenate([m[..., :3, :3].reshape(m.shape[:-2] + (9,)), m[..., :3, 3]], -1)


def _rotation_matrix(q) -> np.ndarray:
    """Unit quaternion (x, y, z, w) -> 3x3, the matrix glTF's node rotation gives."""
    from .gltf import _node_matrix

    return _node_matrix({"rotation": list(q)})[:3, :3]


def subtree_ends(parent) -> np.ndarray:
    """(J) int64: one past the last joint of each joint's subtree, for joints in a depth-first order (parent[k] < k)."""
    parent = np.asarray(parent)
    end = np.arange(1, len(parent) + 1)
    for k in range(len(parent) - 1, -1, -1):
        if parent[k] >= 0:
            end[parent[k]] = max(end[parent[k]], end[k])
    return end


def rig_arrays(rig) -> RigArrays:
    """The host side of a fit: the joints in topological order, every bind and slot renumbered, and the per-joint vertex
    lists, each built once per fit."""
    order = np.asarray(rig.order, np.int64)
    J = len(order)
    pos = np.empty(J, np.int64)
    pos[order] = np.arange(J)
    par = np.asarray(rig.parent, np.int64)[order]
    parent = np.where(par >= 0, pos[np.maximum(par, 0)], -1)
    if (parent >= np.arange(J)).any():
        raise ValueError("rig.order is not a topological order of the joints")
    end = subtree_ends(parent)
    if not all((parent[k + 1:end[k]] >= k).all() for k in range(J)):
        raise ValueError("rig.order is not a depth-first order of the joints")
    above = _xf12(np.asarray(rig.above)[order])
    above_inv = np.zeros((J, 9))
    for k in np.flatnonzero(parent < 0):
        above_inv[k] = np.linalg.inv(above[k, :9].reshape(3, 3)).ravel()
    bind_joint = pos[np.asarray(rig.bind_joint, np.int64)]
    slot_bind = np.asarray(rig.slot_bind, np.int32)
    slot_weight = np.asarray(rig.slot_weight, np.float64)
    V = len(slot_bind)
    used = slot_weight > 0
    cur = np.where(used, bind_joint[slot_bind], -1)
    keys = []
    rows = np.broadcast_to(np.arange(V)[:, None], cur.shape)
    while (cur >= 0).any():
        live = cur >= 0
        keys.append(cur[live] * V + rows[live])
        cur = np.where(live, parent[np.maximum(cur, 0)], -1)
    keys = np.unique(np.concatenate(keys)) if keys else np.zeros(0, np.int64)
    offsets = np.searchsorted(keys, np.arange(J + 1) * V)
    return RigArrays(order=order, parent=parent.astype(np.int32), subtree_end=end, scale=np.asarray(rig.scale)[order].copy(),
                     above=above, above_inv=above_inv, binds=_xf12(rig.binds), bind_joint=bind_joint.astype(np.int32),
                     rotations=np.stack([_rotation_matrix(q).ravel() for q in np.asarray(rig.rotation)[order]]),
                     translations=np.asarray(rig.translation, np.float64)[order].copy(),
                     points=np.asarray(rig.points, np.float64), rest=np.asarray(rig.rest, np.float64),
                     slot_bind=slot_bind, slot_weight=slot_weight, lists=(keys % V).astype(np.int32) if V else keys,
                     offsets=offsets)


def rig_tensors(a: RigArrays, frames: int, device) -> RigTensors:
    cuda = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(device)
    J, NB = len(a.parent), len(a.bind_joint)
    return RigTensors(parent=cuda(a.parent), scale=cuda(a.scale), above=cuda(a.above), above_inv=cuda(a.above_inv),
                      binds=cuda(a.binds), bind_joint=cuda(a.bind_joint), points=cuda(a.points), rest=cuda(a.rest),
                      slot_bind=cuda(a.slot_bind), slot_weight=cuda(a.slot_weight),
                      world=torch.empty(frames, J, 12, dtype=torch.float64, device=device),
                      skin=torch.empty(frames, NB, 12, dtype=torch.float64, device=device),
                      scratch=ops.rig_scratch(frames, len(a.points), device))


def run_sweeps(t: RigTensors, parent, subtree_end, rot: torch.Tensor, trans: torch.Tensor, verts: torch.Tensor,
               joint_lists: list, history: torch.Tensor) -> None:
    """len(history) coordinate-descent sweeps of the state (rot, trans) in place: every joint in order takes its exact
    rotation update over joint_lists[k], then a root its translation update; history[s] (T + 1) receives the error after
    sweep s.  Everything is enqueued, with no host round trip."""
    for s in range(history.shape[0]):
        for k in range(len(parent)):
            end = int(subtree_end[k])
            ops.rig_rotation_update(t, rot, trans, verts, joint_lists[k], k, end)
            if parent[k] < 0:
                ops.rig_translation_update(t, rot, trans, verts, joint_lists[k], k, end)
        ops.rig_error(t, rot, trans, verts, history[s])


def fit_rig_animation(rig, vertices, sweeps: int = DEFAULT_SWEEPS, device: Optional[torch.device] = None) -> RigFit:
    """Fit the local joint rotations and root translations of `rig` (a `gltf.GltfRig`) to the (T, V, 3) animation
    `vertices` (in `load_glb`'s vertex order and frame) -> RigFit.  ValueError: a non-finite value, a shape that does not
    match the rig's vertices, or sweeps < 0."""
    v = np.ascontiguousarray(vertices, dtype=np.float64)
    V = len(rig.rest)
    if v.ndim != 3 or v.shape[0] < 1 or v.shape[1:] != (V, 3):
        raise ValueError(f"vertices must be (T, {V}, 3) with T >= 1 for this rig, got {v.shape}")
    if not np.isfinite(v).all():
        raise ValueError("vertices contain a non-finite value")
    if sweeps < 0:
        raise ValueError(f"sweeps must be >= 0, got {sweeps}")
    T = v.shape[0]
    a = rig_arrays(rig)
    J = len(a.parent)
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(dev):
        t = rig_tensors(a, T, dev)
        verts = torch.from_numpy(v).to(dev)
        rot = torch.from_numpy(np.ascontiguousarray(np.broadcast_to(a.rotations, (T, J, 9)))).to(dev)
        trans = torch.from_numpy(np.ascontiguousarray(np.broadcast_to(a.translations, (T, J, 3)))).to(dev)
        lists = torch.from_numpy(a.lists).to(dev)
        joint_lists = [lists[int(a.offsets[k]):int(a.offsets[k + 1])] for k in range(J)]
        history = torch.empty(sweeps + 1, T + 1, dtype=torch.float64, device=dev)
        ops.rig_error(t, rot, trans, verts, history[0])
        run_sweeps(t, a.parent, a.subtree_end, rot, trans, verts, joint_lists, history[1:])
        frame_errors, max_error2 = ops.rig_error(t, rot, trans, verts)
        rot_pre, trans_pre = rot.cpu().numpy(), trans.cpu().numpy()
        hist = history[:, T].cpu().numpy().tolist()
        total, max2 = float(frame_errors[T]), float(max_error2[0])
    from .gltf import _quaternions

    mats = np.empty_like(rot_pre)
    mats[:, a.order] = rot_pre
    translations = np.empty_like(trans_pre)
    translations[:, a.order] = trans_pre
    mats = mats.reshape(T, J, 3, 3)
    diag = float(np.linalg.norm(a.rest.max(0) - a.rest.min(0)))
    scale = 1.0 / diag if diag > 0 else 1.0
    fit = RigFit(rotations=_quaternions(mats), rotation_matrices=mats, translations=translations, history=hist,
                 rms_error=float(np.sqrt(total / (T * V))) * scale, max_error=float(np.sqrt(max2)) * scale)
    logger.info(f"Rig fit: {J} joints, {T} frames x {V} vertices, {sweeps} sweeps, RMS error {fit.rms_error:.3e} and max "
                f"error {fit.max_error:.3e} of the rest bounding-box diagonal")
    return fit
