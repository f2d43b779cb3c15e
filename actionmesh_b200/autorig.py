"""A skeleton found from the vertex animation itself, its joint rotations and skin weights fitted on the GPU.

    fit = fit_auto_rig(vertices (T, V, 3), faces (F, 3), n_joints)     -> AutoRigFit
    gltf.write_auto_rig_glb(path, fit, faces)

The method follows Le & Deng 2014 ("Robust and accurate skeletal rigging from mesh sequences"); every rule is in
DESIGN.md §22.  Bones and joints share one index j in [0, B):

  1. bones: `skinning.fit_skinning` gives B rigid bones, their transforms [R_j^t | t_j^t], weights and centres c_j.
  2. pair statistics (GPU): face edges whose ends have different dominant bones make the two bones adjacent; the mean
     rest midpoint of those edges is the pair's prior joint point m_ij.
  3. joint solve (GPU): per pair, the point c_ij both bones move alike, argmin sum_t |D_t c - d_t|^2 + LAMBDA T |c - m_ij|^2
     (D_t = R_i^t - R_j^t, d_t = t_j^t - t_i^t), and its cost e_ij = sum_t |D_t c_ij - d_t|^2 / T.
  4. topology (host): Kruskal over the pairs in ascending (not adjacent, e_ij, i, j) gives one tree; the bone of largest
     total weight is the root, child joints sit at their pair's c_ij, the root joint at c_root; joints depth-first.
  5. rig: default local translation c_k - c_parent, identity rotation, inverse bind translate(-c_k): the default pose is
     the rest pose.  The SSDR transforms give a warm start (local rotations R_parent^T R_k, root translation R c + t).
  6. `rounds` rounds of `sweeps` rig sweeps (`rig.run_sweeps`) then one skin-weight update over the rig's skinning
     transforms, the vertex lists rebuilt on the device.  Every step minimises its own variables, so `history` does not
     increase beyond rounding.
"""
from __future__ import annotations

import logging
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from . import ops, rig, skinning

logger = logging.getLogger(__name__)

LAMBDA = 1e-4          # prior weight per frame, dimensionless (DESIGN.md §22)
DEFAULT_ROUNDS = 4
DEFAULT_SWEEPS = 10


@dataclass
class AutoRigFit:
    """A found skeleton and its animation, joints in the file's depth-first order: parent (J) int64 (-1 for joint 0, the
    root) and bones (J), the SSDR bone behind each joint; positions (J, 3) fp64, the rest joint positions; rotations
    (T, J, 4) unit quaternions (x, y, z, w) and rotation_matrices (T, J, 3, 3), the local rotations; root_translations
    (T, 3), the root joint's translation; rest (V, 3); joints (V, 4) int32 and weights (V, 4) fp64 (unused slots 0 / 0);
    history: sum_t,i |v^ - v|^2 after the warm start and after every half round; rms_error and max_error: the final RMS and
    largest |v^ - v|, and ssdr_rms_error the flat bones' RMS, each relative to the rest bounding-box diagonal."""
    parent: np.ndarray
    bones: np.ndarray
    positions: np.ndarray
    rotations: np.ndarray
    rotation_matrices: np.ndarray
    root_translations: np.ndarray
    rest: np.ndarray
    joints: np.ndarray
    weights: np.ndarray
    history: list
    rms_error: float
    max_error: float
    ssdr_rms_error: float


def pair_index(i: int, j: int, n_bones: int) -> int:
    """The pair of bones i < j in lexicographic order."""
    return i * (2 * n_bones - i - 1) // 2 + (j - i - 1)


def skeleton_topology(pair_count, pair_cost, bone_weight) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """The tree over B bones from the pair tables (P = B (B - 1) / 2, lexicographic pairs) and each bone's total weight
    -> (bones (J): the bone of each joint in depth-first order from the root, children in ascending bone index; parent (J):
    the parent joint, -1 for the root; pair (J): the pair of each joint's tree edge, -1 for the root).  Kruskal takes the
    pairs in ascending (not adjacent, cost, i, j); the root is the bone of largest total weight, ties to the lower index."""
    w = np.asarray(bone_weight, np.float64)
    B = len(w)
    i, j = np.triu_indices(B, 1)
    count, cost = np.asarray(pair_count), np.asarray(pair_cost, np.float64)
    if len(count) != len(i) or len(cost) != len(i):
        raise ValueError(f"pair tables must hold {len(i)} pairs for {B} bones")
    root_of = np.arange(B)

    def find(x: int) -> int:
        while root_of[x] != x:
            root_of[x] = root_of[root_of[x]]
            x = root_of[x]
        return x

    adj: list = [[] for _ in range(B)]
    for p in np.lexsort((j, i, cost, count <= 0)):
        a, b = find(int(i[p])), find(int(j[p]))
        if a != b:
            root_of[max(a, b)] = min(a, b)
            adj[int(i[p])].append((int(j[p]), int(p)))
            adj[int(j[p])].append((int(i[p]), int(p)))
    root = int(np.argmax(w))
    bones, parent, pair = [], [], []
    stack = [(root, -1, -1)]
    while stack:
        b, par, p = stack.pop()
        k = len(bones)
        bones.append(b)
        parent.append(par)
        pair.append(p)
        for c, q in sorted(adj[b], reverse=True):
            if c != (bones[par] if par >= 0 else -1):
                stack.append((c, k, q))
    return np.asarray(bones, np.int64), np.asarray(parent, np.int64), np.asarray(pair, np.int64)


def _mat3_t_mul(A: np.ndarray, Bm: np.ndarray) -> np.ndarray:
    """(..., 9) row-major A^T B, each entry ((A_0a B_0b + A_1a B_1b) + A_2a B_2b)."""
    return np.stack([(A[..., a] * Bm[..., b] + A[..., 3 + a] * Bm[..., 3 + b]) + A[..., 6 + a] * Bm[..., 6 + b]
                     for a in range(3) for b in range(3)], -1)


def rig_start(bones, parent, positions, transforms) -> tuple[np.ndarray, np.ndarray]:
    """The warm start from the SSDR transforms (T, B, 12) -> (rotations (T, J, 9), translations (T, J, 3)): local
    R_parent^T R_k (R_root for the root), c_k - c_parent for every other joint's translation and, for the root,
    ((R_0 c_0 + R_1 c_1) + R_2 c_2) + t per row of R_root c_root + t_root."""
    xf = np.asarray(transforms, np.float64)[:, bones]
    T, J = xf.shape[:2]
    rot = np.empty((T, J, 9))
    trans = np.empty((T, J, 3))
    c = np.asarray(positions, np.float64)
    for k in range(J):
        p = parent[k]
        rot[:, k] = xf[:, k, :9] if p < 0 else _mat3_t_mul(xf[:, p, :9], xf[:, k, :9])
        trans[:, k] = c[k] - c[p] if p >= 0 else 0.0
    R, t0 = xf[:, 0, :9], xf[:, 0, 9:]
    trans[:, 0] = np.stack([((R[:, 3 * a] * c[0, 0] + R[:, 3 * a + 1] * c[0, 1]) + R[:, 3 * a + 2] * c[0, 2]) + t0[:, a]
                            for a in range(3)], -1)
    return rot, trans


def rig_layout(parent, positions, rest) -> rig.RigArrays:
    """The kernels' layout of the found skeleton (joints already depth-first): one bind per joint, translate(-c_k); the
    slots and vertex lists are left empty (the fit fills them on the device)."""
    parent = np.asarray(parent, np.int64)
    J, V = len(parent), len(rest)
    end = rig.subtree_ends(parent)
    c = np.asarray(positions, np.float64)
    eye12 = np.tile(np.array([1.0, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0]), (J, 1))
    binds = eye12.copy()
    binds[:, 9:] = -c
    above, above_inv = np.zeros((J, 12)), np.zeros((J, 9))
    above[0], above_inv[0] = eye12[0], eye12[0, :9]
    trans = np.array([c[k] - c[parent[k]] if parent[k] >= 0 else c[k] for k in range(J)]).reshape(J, 3)
    return rig.RigArrays(order=np.arange(J), parent=parent.astype(np.int32), subtree_end=end, scale=np.ones((J, 3)),
                         above=above, above_inv=above_inv, binds=binds, bind_joint=np.arange(J, dtype=np.int32),
                         rotations=eye12[:, :9].copy(), translations=trans, points=np.asarray(rest, np.float64),
                         rest=np.asarray(rest, np.float64), slot_bind=np.zeros((V, 8), np.int32),
                         slot_weight=np.zeros((V, 8)), lists=np.zeros(0, np.int32), offsets=np.zeros(J + 1, np.int64))


def list_capacity(parent, n_vertices: int) -> int:
    """An upper bound of the lists' total length: every vertex is listed under the ancestors of its <= 4 joints."""
    parent = np.asarray(parent)
    depth = np.zeros(len(parent), np.int64)
    for k in range(1, len(parent)):
        depth[k] = depth[parent[k]] + 1
    return int(n_vertices) * int(min(len(parent), 4 * (int(depth.max()) + 1)))


def _check(v: np.ndarray, f: np.ndarray, n_joints: int, rounds: int, sweeps: int) -> None:
    if v.ndim != 3 or v.shape[2] != 3 or v.shape[0] < 1 or v.shape[1] < 1:
        raise ValueError(f"vertices must be (T, V, 3) with T >= 1 and V >= 1, got {v.shape}")
    if not np.isfinite(v).all():
        raise ValueError("vertices contain a non-finite value")
    V = v.shape[1]
    if f.ndim != 2 or f.shape[1] != 3 or len(f) < 1:
        raise ValueError(f"faces must be (F, 3) with F >= 1, got {f.shape}")
    if f.min() < 0 or f.max() >= V:
        raise ValueError(f"faces index outside the {V} vertices")
    n_max = min(V, skinning.MAX_BONES)
    if not 1 <= n_joints <= n_max:
        raise ValueError(f"n_joints must be in [1, {n_max}] for {V} vertices, got {n_joints}")
    if rounds < 0 or sweeps < 0:
        raise ValueError(f"rounds and sweeps must be >= 0, got {rounds} and {sweeps}")


@dataclass
class AutoRigState:
    """A fit in progress, on the device, joints depth-first: the found skeleton (bones, parent, positions, the SSDR fit and
    its pair tables on the host), the rig's layout `a` and tensors `t`, the state rot (T, J, 9) / trans (T, J, 3) /
    joints / weights (V, 4), the animation, and the per-joint vertex lists of the current slots."""
    sk: skinning.SkinningFit
    pair_count: np.ndarray
    pair_joint: np.ndarray
    pair_cost: np.ndarray
    bone_weight: np.ndarray
    bones: np.ndarray
    parent: np.ndarray
    positions: np.ndarray
    a: rig.RigArrays
    t: rig.RigTensors
    verts: torch.Tensor
    rest: torch.Tensor
    rot: torch.Tensor
    trans: torch.Tensor
    joints: torch.Tensor
    weights: torch.Tensor
    subtree_end: torch.Tensor
    lists: torch.Tensor
    offsets: torch.Tensor
    list_scratch: torch.Tensor
    joint_lists: list


def refresh_lists(st: AutoRigState) -> None:
    """The rig's slots from (joints, weights) and the per-joint vertex lists from the slots, on the device; the J + 1
    offsets are read back to size the next sweeps' launches."""
    J = len(st.parent)
    ops.autorig_slots(st.joints, st.weights, st.t.slot_bind, st.t.slot_weight)
    ops.autorig_joint_lists(st.t, st.subtree_end, st.lists, st.offsets, st.list_scratch)
    off = st.offsets.cpu().numpy()
    if off[J] > len(st.lists):
        raise RuntimeError(f"joint lists need {off[J]} entries, more than the bound {len(st.lists)}")
    st.joint_lists = [st.lists[int(off[k]):int(off[k + 1])] for k in range(J)]


def start_auto_rig(v: np.ndarray, f: np.ndarray, B: int, dev: torch.device) -> AutoRigState:
    """Steps 1-6 of the fit (checked float64 vertices, int32 faces; `dev` current): SSDR bones, pair statistics, joint
    solve, topology, the skeleton's layout and the warm start, then the slots and lists."""
    T, V, _ = v.shape
    sk = skinning.fit_skinning(v, B, device=dev)
    cuda = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)  # noqa: E731
    verts = cuda(v)
    rest = verts[0].contiguous()
    xf = np.concatenate([sk.rotations.reshape(T, B, 9), sk.translations], -1)
    count, prior = ops.autorig_pair_stats(rest, cuda(f), cuda(sk.joints), cuda(sk.weights), B)
    totals = ops.autorig_bone_weights(cuda(sk.joints), cuda(sk.weights), B)
    pair_joint, pair_cost = ops.autorig_joint_solve(cuda(xf), cuda(sk.centres), count, prior, LAMBDA)
    count_h, cost_h, totals_h, pj = (x.cpu().numpy() for x in (count, pair_cost, totals, pair_joint))
    bones, parent, pair = skeleton_topology(count_h, cost_h, totals_h)
    positions = np.stack([pj[p] if p >= 0 else sk.centres[b] for b, p in zip(bones, pair)])
    pos = np.empty(B, np.int64)
    pos[bones] = np.arange(B)
    a = rig_layout(parent, positions, v[0])
    rot0, trans0 = rig_start(bones, parent, positions, xf)
    st = AutoRigState(sk=sk, pair_count=count_h, pair_joint=pj, pair_cost=cost_h, bone_weight=totals_h, bones=bones,
                      parent=parent, positions=positions, a=a, t=rig.rig_tensors(a, T, dev), verts=verts, rest=rest,
                      rot=cuda(rot0), trans=cuda(trans0),
                      joints=cuda(np.where(sk.weights > 0, pos[sk.joints], 0).astype(np.int32)), weights=cuda(sk.weights),
                      subtree_end=cuda(a.subtree_end.astype(np.int32)),
                      lists=torch.empty(list_capacity(parent, V), dtype=torch.int32, device=dev),
                      offsets=torch.empty(B + 1, dtype=torch.int32, device=dev),
                      list_scratch=ops.autorig_list_scratch(V, B, dev), joint_lists=[])
    refresh_lists(st)
    return st


def sweep_half(st: AutoRigState, sweeps: int) -> None:
    """The first half of a round: `sweeps` rig sweeps of (rot, trans)."""
    errors = torch.empty(sweeps, st.verts.shape[0] + 1, dtype=torch.float64, device=st.verts.device)
    rig.run_sweeps(st.t, st.a.parent, st.a.subtree_end, st.rot, st.trans, st.verts, st.joint_lists, errors)


def weight_half(st: AutoRigState) -> None:
    """The second half of a round: the skin weights refitted over the rig's skinning transforms K = G B, then the slots
    and lists rebuilt."""
    ops.rig_forward(st.t, st.rot, st.trans)
    _, _, cand = ops.skin_rigid_error(st.rest, st.verts, st.t.skin)
    ops.skin_weight_update(st.rest, st.verts, st.t.skin, cand, st.joints, st.weights)
    refresh_lists(st)


def fit_auto_rig(vertices, faces, n_joints: int, rounds: int = DEFAULT_ROUNDS, sweeps: int = DEFAULT_SWEEPS,
                 device: Optional[torch.device] = None) -> AutoRigFit:
    """Find a skeleton of `n_joints` joints for the (T, V, 3) animation `vertices` on (F, 3) `faces` (rest pose
    vertices[0]) and fit its joint rotations, root translation and skin weights -> AutoRigFit.  ValueError: a non-finite
    value, T < 1, no faces or a face index out of range, n_joints outside [1, min(V, 256)], or rounds / sweeps < 0."""
    v = np.ascontiguousarray(vertices, dtype=np.float64)
    f = np.ascontiguousarray(np.asarray(faces).reshape(-1, 3) if np.asarray(faces).size else np.zeros((0, 3)))
    _check(v, f, int(n_joints), int(rounds), int(sweeps))
    J = int(n_joints)
    T, V, _ = v.shape
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(dev):
        st = start_auto_rig(v, f.astype(np.int32), J, dev)
        history = torch.empty(2 * rounds + 1, T + 1, dtype=torch.float64, device=dev)
        ops.rig_error(st.t, st.rot, st.trans, st.verts, history[0])
        for r in range(rounds):
            sweep_half(st, sweeps)
            ops.rig_error(st.t, st.rot, st.trans, st.verts, history[2 * r + 1])
            weight_half(st)
            ops.rig_error(st.t, st.rot, st.trans, st.verts, history[2 * r + 2])
        frame_errors, max_error2 = ops.rig_error(st.t, st.rot, st.trans, st.verts)
        rot_h, trans_h = st.rot.cpu().numpy(), st.trans.cpu().numpy()
        joints_h, weights_h = st.joints.cpu().numpy(), st.weights.cpu().numpy()
        hist = history[:, T].cpu().numpy().tolist()
        total, max2 = float(frame_errors[T]), float(max_error2[0])
    from .gltf import _quaternions

    mats = rot_h.reshape(T, J, 3, 3)
    diag = float(np.linalg.norm(v[0].max(0) - v[0].min(0)))
    scale = 1.0 / diag if diag > 0 else 1.0
    fit = AutoRigFit(parent=st.parent, bones=st.bones, positions=st.positions, rotations=_quaternions(mats),
                     rotation_matrices=mats, root_translations=trans_h[:, 0].copy(), rest=v[0].copy(), joints=joints_h,
                     weights=weights_h, history=hist, rms_error=float(np.sqrt(total / (T * V))) * scale,
                     max_error=float(np.sqrt(max2)) * scale, ssdr_rms_error=st.sk.rms_error)
    logger.info(f"Auto rig: {J} joints, {T} frames x {V} vertices, {rounds} rounds of {sweeps} sweeps, RMS error "
                f"{fit.rms_error:.3e} (flat bones {fit.ssdr_rms_error:.3e}) and max error {fit.max_error:.3e} of the rest "
                f"bounding-box diagonal")
    return fit


def posed_vertices(fit: AutoRigFit) -> np.ndarray:
    """(T, V, 3) v^ of a fit by linear blend skinning in float64 (numpy matrix products): G_k = G_parent [R_k | c_k -
    c_parent], the root [R_root | tau], K_k = G_k translate(-c_k)."""
    T, J = fit.rotation_matrices.shape[:2]
    G = np.zeros((T, J, 4, 4))
    G[:, :, 3, 3] = 1.0
    for k in range(J):
        local = np.zeros((T, 4, 4))
        local[:, :3, :3] = fit.rotation_matrices[:, k]
        local[:, 3, 3] = 1.0
        p = fit.parent[k]
        local[:, :3, 3] = fit.root_translations if p < 0 else fit.positions[k] - fit.positions[p]
        G[:, k] = local if p < 0 else G[:, p] @ local
    K = G.copy()
    K[:, :, :3, 3] -= np.einsum("tkij,kj->tki", G[:, :, :3, :3], fit.positions)
    Kv = K[:, fit.joints]                                                       # (T, V, 4, 4, 4)
    u = np.einsum("tvsij,vj->tvsi", Kv[..., :3, :3], fit.rest) + Kv[..., :3, 3]
    return np.einsum("vs,tvsi->tvi", fit.weights, u)
