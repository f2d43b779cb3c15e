"""numpy float64 restatement of csrc/autorig.cu and of the whole automatic-rig fit (DESIGN.md §22), written from the rules.

Every product, sum, quotient and square root is one numpy float64 operation (round to nearest, never fused), in the
kernels' order, so the results equal the GPU's bit for bit.  The SSDR bones come from skinning_ref and the rig sweeps and
errors from rig_ref; this file states only what §22 adds.
"""
from __future__ import annotations

from types import SimpleNamespace

import numpy as np

import rig_ref
import skinning_ref

LAMBDA = 1e-4
TILE = 256


def pair_index(i, j, B):
    return i * (2 * B - i - 1) // 2 + (j - i - 1)


def dominant(joints, weights) -> np.ndarray:
    """The used slot of largest weight, ties to the earlier slot; -1 without a used slot."""
    V = len(weights)
    best, bw = np.full(V, -1), np.zeros(V)
    for k in range(4):
        take = (weights[:, k] > 0) & ((best < 0) | (weights[:, k] > bw))
        best = np.where(take, joints[:, k], best)
        bw = np.where(take, weights[:, k], bw)
    return best


def pair_stats(rest, faces, joints, weights, B):
    """-> (pair_count (P) int32, pair_prior (P, 3)): edges in edge order 3f + k, (f_k, f_(k+1) mod 3)."""
    P = B * (B - 1) // 2
    dom = dominant(joints, weights)
    a = faces.reshape(-1)
    b = faces[:, [1, 2, 0]].reshape(-1)
    da, db = dom[a], dom[b]
    cross = (da >= 0) & (db >= 0) & (da != db)
    lo, hi = np.minimum(da, db), np.maximum(da, db)
    key = np.where(cross, pair_index(lo, hi, B), -1)
    count = np.zeros(P, np.int32)
    s = np.zeros((P, 3))
    mid = (rest[a] + rest[b]) * 0.5
    for e in np.flatnonzero(cross):                    # edge order
        count[key[e]] += 1
        s[key[e]] = s[key[e]] + mid[e]
    prior = np.where(count[:, None] > 0, s / np.maximum(count, 1)[:, None].astype(np.float64), 0.0)
    return count, prior


def bone_weights(joints, weights, B) -> np.ndarray:
    """Per 256-vertex tile in vertex then slot order, then the tiles in order."""
    V = len(weights)
    tiles = -(-V // TILE)
    parts = np.zeros((tiles, B))
    for t in range(tiles):
        for v in range(t * TILE, min(V, (t + 1) * TILE)):
            for k in range(4):
                if weights[v, k] > 0:
                    parts[t, joints[v, k]] = parts[t, joints[v, k]] + weights[v, k]
    return skinning_ref.sum_in_order(parts)


def joint_solve(xf, centres, count, prior, lam=LAMBDA):
    """-> (pair_joint (P, 3), pair_cost (P)); xf (T, B, 12)."""
    T, B = xf.shape[:2]
    i, j = np.triu_indices(B, 1)
    P = len(i)
    N = np.zeros((P, 6))
    r = np.zeros((P, 3))
    Xi, Xj = xf[:, i], xf[:, j]                        # (T, P, 12)
    D = Xi[..., :9] - Xj[..., :9]
    d = Xj[..., 9:] - Xi[..., 9:]
    idx = [(a, b) for a in range(3) for b in range(a, 3)]
    for t in range(T):
        for q, (a, b) in enumerate(idx):
            N[:, q] = N[:, q] + ((D[t, :, a] * D[t, :, b] + D[t, :, 3 + a] * D[t, :, 3 + b]) + D[t, :, 6 + a] * D[t, :, 6 + b])
        for a in range(3):
            r[:, a] = r[:, a] + ((D[t, :, a] * d[t, :, 0] + D[t, :, 3 + a] * d[t, :, 1]) + D[t, :, 6 + a] * d[t, :, 2])
    m = np.where(count[:, None] > 0, prior, (centres[i] + centres[j]) * 0.5)
    lt = lam * float(T)
    a00, a11, a22 = N[:, 0] + lt, N[:, 3] + lt, N[:, 5] + lt
    b0, b1, b2 = r[:, 0] + lt * m[:, 0], r[:, 1] + lt * m[:, 1], r[:, 2] + lt * m[:, 2]
    l00 = np.sqrt(a00)
    l10, l20 = N[:, 1] / l00, N[:, 2] / l00
    l11 = np.sqrt(a11 - l10 * l10)
    l21 = (N[:, 4] - l20 * l10) / l11
    l22 = np.sqrt((a22 - l20 * l20) - l21 * l21)
    y0 = b0 / l00
    y1 = (b1 - l10 * y0) / l11
    y2 = ((b2 - l20 * y0) - l21 * y1) / l22
    c2 = y2 / l22
    c1 = (y1 - l21 * c2) / l11
    c0 = ((y0 - l10 * c1) - l20 * c2) / l00
    e = np.zeros(P)
    for t in range(T):
        res = [((D[t, :, 3 * a] * c0 + D[t, :, 3 * a + 1] * c1) + D[t, :, 3 * a + 2] * c2) - d[t, :, a] for a in range(3)]
        e = e + ((res[0] * res[0] + res[1] * res[1]) + res[2] * res[2])
    return np.stack([c0, c1, c2], -1), e / float(T)


def slots(joints, weights):
    """(V, 4) -> (slot_bind (V, 8) int32, slot_weight (V, 8)), used slots first."""
    V = len(weights)
    sb, sw = np.zeros((V, 8), np.int32), np.zeros((V, 8))
    for v in range(V):
        used = [k for k in range(4) if weights[v, k] > 0]
        sb[v, :len(used)] = joints[v, used]
        sw[v, :len(used)] = weights[v, used]
    return sb, sw


def joint_lists(bind_joint, slot_bind, slot_weight, subtree_end):
    """-> (lists, offsets (J + 1)): joint k's vertices with a used slot in its subtree, ascending, joint after joint."""
    jb = np.where(slot_weight > 0, np.asarray(bind_joint)[slot_bind], -1)
    lists, offsets = [], [0]
    for k in range(len(subtree_end)):
        inside = ((jb >= k) & (jb < subtree_end[k])).any(1)
        lists.append(np.flatnonzero(inside))
        offsets.append(offsets[-1] + int(inside.sum()))
    return np.concatenate(lists).astype(np.int32), np.asarray(offsets, np.int64)


def topology(count, cost, totals):
    """Kruskal in ascending (not adjacent, cost, i, j); root = largest total (lower index on ties); depth-first, children
    in ascending bone order -> (bones, parent, pair)."""
    B = len(totals)
    i, j = np.triu_indices(B, 1)
    comp = list(range(B))
    edges = []
    for p in sorted(range(len(i)), key=lambda p: (count[p] <= 0, cost[p], i[p], j[p])):
        ca, cb = comp[i[p]], comp[j[p]]
        if ca != cb:
            comp = [ca if c == cb else c for c in comp]
            edges.append((int(i[p]), int(j[p]), p))
    root = max(range(B), key=lambda b: (totals[b], -b))
    bones, parent, pair = [], [], []

    def visit(b, par, p):
        k = len(bones)
        bones.append(b)
        parent.append(par)
        pair.append(p)
        nb = sorted([(y, q) for x, y, q in edges if x == b] + [(x, q) for x, y, q in edges if y == b])
        for c, q in nb:
            if par < 0 or c != bones[par]:
                visit(c, k, q)

    visit(root, -1, -1)
    return np.array(bones), np.array(parent), np.array(pair)


def warm_start(xf, bones, parent, c):
    """-> (rotations (T, J, 9), translations (T, J, 3)): local R_parent^T R_k (R_root for the root), c_k - c_parent, and
    the root's R c + t (apply_xf)."""
    X = xf[:, bones]
    T, J = X.shape[:2]
    rot = np.empty((T, J, 9))
    trans = np.empty((T, J, 3))
    for k in range(J):
        p = parent[k]
        if p < 0:
            rot[:, k] = X[:, k, :9]
        else:
            A, Bm = X[:, p, :9], X[:, k, :9]
            rot[:, k] = np.stack([(A[:, a] * Bm[:, b] + A[:, 3 + a] * Bm[:, 3 + b]) + A[:, 6 + a] * Bm[:, 6 + b]
                                  for a in range(3) for b in range(3)], -1)
            trans[:, k] = c[k] - c[p]
    trans[:, 0] = skinning_ref.apply_xf(X[:, 0], c[0])
    return rot, trans


def fit(vertices, faces, B, rounds, sweeps, iterations=20):
    """The whole fit -> dict of parent, bones, positions, rotations (T, J, 9), translations (T, J, 3), joints, weights,
    history."""
    v = np.asarray(vertices, np.float64)
    T, V, _ = v.shape
    rest = v[0]
    sk = skinning_ref.fit(v, B, iterations)
    xf, sj, sw, centres = sk["transforms"], sk["joints"], sk["weights"], sk["centres"]
    count, prior = pair_stats(rest, faces, sj, sw, B)
    totals = bone_weights(sj, sw, B)
    pj, cost = joint_solve(xf, centres, count, prior)
    bones, parent, pair = topology(count, cost, totals)
    J = B
    c = np.stack([pj[p] if p >= 0 else centres[b] for b, p in zip(bones, pair)])
    pos = np.empty(B, np.int64)
    pos[bones] = np.arange(J)
    end = np.arange(1, J + 1)
    for k in range(J - 1, 0, -1):
        end[parent[k]] = max(end[parent[k]], end[k])
    binds = np.tile(np.array([1.0, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0]), (J, 1))
    binds[:, 9:] = -c
    above = np.zeros((J, 12))
    above[0] = [1.0, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0]
    above_inv = np.zeros((J, 9))
    above_inv[0] = above[0, :9]
    a = SimpleNamespace(parent=parent, scale=np.ones((J, 3)), above=above, above_inv=above_inv, binds=binds,
                        bind_joint=np.arange(J), points=rest, rest=rest, subtree_end=end)
    rot, trans = warm_start(xf, bones, parent, c)
    joints = np.where(sw > 0, pos[sj], 0).astype(np.int32)
    weights = sw.copy()

    def refresh():
        a.slot_bind, a.slot_weight = slots(joints, weights)
        a.lists, a.offsets = joint_lists(a.bind_joint, a.slot_bind, a.slot_weight, end)

    refresh()
    history = [rig_ref.error(a, rot, trans, v)[0][T]]
    for _ in range(rounds):
        for _ in range(sweeps):
            for k in range(J):
                lst = rig_ref.joint_list(a, k)
                rot = rig_ref.rotation_update(a, rot, trans, v, lst, k, int(end[k]))
                if parent[k] < 0:
                    trans = rig_ref.translation_update(a, rot, trans, v, lst, k, int(end[k]))
        history.append(rig_ref.error(a, rot, trans, v)[0][T])
        _, skin = rig_ref.forward(a, rot, trans)
        _, _, cand = skinning_ref.rigid_error(rest, v, skin)
        joints, weights = skinning_ref.weight_update(rest, v, skin, cand, joints, weights)
        refresh()
        history.append(rig_ref.error(a, rot, trans, v)[0][T])
    return dict(rig=a, parent=parent, bones=bones, positions=c, rotations=rot, translations=trans, joints=joints,
                weights=weights, history=history, pair_count=count, pair_prior=prior, pair_joint=pj, pair_cost=cost,
                totals=totals, ssdr=sk)
