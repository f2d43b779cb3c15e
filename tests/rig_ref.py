"""numpy float64 restatement of csrc/rig.cu (DESIGN.md §21), written from the rules and not from actionmesh_b200/rig.py.

Every product, sum, quotient and square root is one numpy float64 operation (round to nearest, never fused), in the kernels'
order; sums run in the kernels' fixed orders (skinning_ref's per-tile halving trees, tiles in order, frames in order), so
the results equal the GPU's bit for bit.  The layouts are `rig.RigArrays`' (joints in topological order, transforms as 12
doubles: L row-major then t): rotations (T, J, 9), translations (T, J, 3), world (T, J, 12), skin (T, NB, 12).
"""
from __future__ import annotations

import numpy as np

from skinning_ref import apply_xf, horn_rotation, norm2, sum_in_order, tile_partials

SLOTS = 8


def compose(A: np.ndarray, B: np.ndarray) -> np.ndarray:
    """(..., 12) o (..., 12): linear ((A_a0 B_0b + A_a1 B_1b) + A_a2 B_2b), translation apply_xf(A, t_B)."""
    lin = [(A[..., 3 * a] * B[..., b] + A[..., 3 * a + 1] * B[..., 3 + b]) + A[..., 3 * a + 2] * B[..., 6 + b]
           for a in range(3) for b in range(3)]
    return np.concatenate([np.stack(lin, -1), apply_xf(A, B[..., 9:12])], -1)


def forward(a, rotations: np.ndarray, translations: np.ndarray):
    """-> (world (T, J, 12), skin (T, NB, 12)): joints in order, local = [R_ab s_b | tau], G = P o local."""
    T, J = rotations.shape[:2]
    world = np.zeros((T, J, 12))
    for j in range(J):
        local = np.concatenate([rotations[:, j] * np.tile(a.scale[j], 3), translations[:, j]], -1)
        P = world[:, a.parent[j]] if a.parent[j] >= 0 else np.broadcast_to(a.above[j], (T, 12))
        world[:, j] = compose(P, local)
    skin = compose(world[:, a.bind_joint], np.broadcast_to(a.binds, (T,) + a.binds.shape))
    return world, skin


def parent_xf(a, world: np.ndarray, j: int) -> np.ndarray:
    """(T, 12) P_j."""
    return world[:, a.parent[j]] if a.parent[j] >= 0 else np.broadcast_to(a.above[j], (world.shape[0], 12))


def blend(a, skin_t: np.ndarray, idx: np.ndarray, j0: int, j1: int):
    """Vertices idx in one frame -> (sub, rest, all (n, 3), m (n,)): slot order from 0, sub / m over slots whose joint is
    in [j0, j1)."""
    n = len(idx)
    sub, rst, al, m = np.zeros((n, 3)), np.zeros((n, 3)), np.zeros((n, 3)), np.zeros(n)
    p = a.points[idx]
    for k in range(SLOTS):
        w = a.slot_weight[idx, k]
        used = w > 0
        b = np.where(used, a.slot_bind[idx, k], 0)
        jb = a.bind_joint[b]
        wu = w[:, None] * apply_xf(skin_t[b], p)
        ins = used & (jb >= j0) & (jb < j1)
        out = used & ~ins
        al = np.where(used[:, None], al + wu, al)
        sub = np.where(ins[:, None], sub + wu, sub)
        m = np.where(ins, m + w, m)
        rst = np.where(out[:, None], rst + wu, rst)
    return sub, rst, al, m


def rotation_update(a, rotations, translations, verts, lst, joint: int, end: int) -> np.ndarray:
    """-> rotations after the rotation update of `joint` (unchanged when `lst` is empty)."""
    rotations = rotations.copy()
    if len(lst) == 0:
        return rotations
    T = rotations.shape[0]
    world, skin = forward(a, rotations, translations)
    P = parent_xf(a, world, joint)
    f = apply_xf(P, translations[:, joint])
    for t in range(T):
        sub, rst, _, m = blend(a, skin[t], lst, joint, end)
        v = verts[t][lst]
        d = sub - m[:, None] * f[t]
        e = (v - rst) - m[:, None] * f[t]
        c = (d[:, :, None] * e[:, None, :]).reshape(-1, 9)
        Hw = sum_in_order(tile_partials(c))
        L, R = P[t, :9], rotations[t, joint]
        X = np.array([(Hw[3 * i] * L[k] + Hw[3 * i + 1] * L[3 + k]) + Hw[3 * i + 2] * L[6 + k]
                      for i in range(3) for k in range(3)])
        Y = np.array([(L[i] * X[k] + L[3 + i] * X[3 + k]) + L[6 + i] * X[6 + k] for i in range(3) for k in range(3)])
        H = np.array([(R[i] * Y[k] + R[3 + i] * Y[3 + k]) + R[6 + i] * Y[6 + k] for i in range(3) for k in range(3)])
        rotations[t, joint] = horn_rotation(H.reshape(1, 3, 3))[0]
    return rotations


def translation_update(a, rotations, translations, verts, lst, joint: int, end: int) -> np.ndarray:
    """-> translations after the translation update of root `joint`."""
    translations = translations.copy()
    if len(lst) == 0:
        return translations
    _, skin = forward(a, rotations, translations)
    Ai = a.above_inv[joint]
    for t in range(rotations.shape[0]):
        _, _, al, m = blend(a, skin[t], lst, joint, end)
        r = verts[t][lst] - al
        c = np.stack([m * m, m * r[:, 0], m * r[:, 1], m * r[:, 2]], -1)
        s = sum_in_order(tile_partials(c))
        if not s[0] > 0:
            continue
        dl = s[1:] / s[0]
        tau = translations[t, joint]
        translations[t, joint] = [tau[i] + ((Ai[3 * i] * dl[0] + Ai[3 * i + 1] * dl[1]) + Ai[3 * i + 2] * dl[2])
                                  for i in range(3)]
    return translations


def posed(a, rotations, translations) -> np.ndarray:
    """(T, V, 3) v^: blended over the used slots, rest for static vertices."""
    _, skin = forward(a, rotations, translations)
    idx = np.arange(len(a.points))
    static = ~(a.slot_weight[:, 0] > 0)
    return np.stack([np.where(static[:, None], a.rest, blend(a, skin[t], idx, 0, 0)[2]) for t in range(len(skin))])


def error(a, rotations, translations, verts):
    """-> (frame errors (T + 1): per frame then the sum in frame order, max |v^ - v|^2)."""
    T = verts.shape[0]
    d2 = norm2(posed(a, rotations, translations) - verts)
    fe = np.zeros(T + 1)
    for t in range(T):
        fe[t] = sum_in_order(tile_partials(d2[t]))
    fe[T] = sum_in_order(fe[:T])
    return fe, float(d2.max())


def joint_list(a, k: int) -> np.ndarray:
    return a.lists[a.offsets[k]:a.offsets[k + 1]]


def fit(a, verts, sweeps: int):
    """The whole fit (DESIGN.md §21) -> (rotations, translations, history), joints in topological order."""
    T, J = verts.shape[0], len(a.parent)
    rot = np.ascontiguousarray(np.broadcast_to(a.rotations, (T, J, 9)))
    trans = np.ascontiguousarray(np.broadcast_to(a.translations, (T, J, 3)))
    history = [error(a, rot, trans, verts)[0][T]]
    for _ in range(sweeps):
        for k in range(J):
            lst = joint_list(a, k)
            rot = rotation_update(a, rot, trans, verts, lst, k, int(a.subtree_end[k]))
            if a.parent[k] < 0:
                trans = translation_update(a, rot, trans, verts, lst, k, int(a.subtree_end[k]))
        history.append(error(a, rot, trans, verts)[0][T])
    return rot, trans, history
