"""numpy float64 restatement of csrc/skinning.cu (DESIGN.md §20), written from the rules and not from actionmesh_b200/skinning.py.

Every product, sum, quotient and square root is one numpy float64 operation (round to nearest, never fused), in the kernels'
order; sums run in the kernels' fixed orders (per-tile halving trees over 32 lanes then 8 warps, then tiles in order), so the
results equal the GPU's bit for bit.  Layouts are the kernels': rest (V, 3), vertices (T, V, 3), transforms (T, B, 12) = R
row-major then t, joints (V, 4) int32 and weights (V, 4), a slot being used when its weight is > 0.
"""
from __future__ import annotations

import itertools

import numpy as np

TILE, LANES, WARPS = 256, 32, 8
N_CAND = 8
SWEEPS = 10
DET_MIN = 1e-12
CLUSTER_ROUNDS = 5
PAIRS = ((0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3))


def apply_xf(m: np.ndarray, p: np.ndarray) -> np.ndarray:
    """u_a = ((R_a0 p_x + R_a1 p_y) + R_a2 p_z) + t_a; m (..., 12), p (..., 3)."""
    return np.stack([((m[..., 3 * a] * p[..., 0] + m[..., 3 * a + 1] * p[..., 1]) + m[..., 3 * a + 2] * p[..., 2]) + m[..., 9 + a]
                     for a in range(3)], -1)


def norm2(r: np.ndarray) -> np.ndarray:
    return (r[..., 0] * r[..., 0] + r[..., 1] * r[..., 1]) + r[..., 2] * r[..., 2]


def dot3(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def blend(xf_t: np.ndarray, joints: np.ndarray, weights: np.ndarray, p: np.ndarray, skip: int = -1) -> np.ndarray:
    """sum over the used slots in slot order whose joint is not `skip` of w u, from 0."""
    s = np.zeros_like(p)
    for k in range(4):
        w, j = weights[:, k], joints[:, k]
        use = (w > 0) & (j != skip)
        u = apply_xf(xf_t[np.where(use, j, 0)], p)
        s = np.where(use[:, None], s + w[:, None] * u, s)
    return s


def _halve(x: np.ndarray, axis: int) -> np.ndarray:
    x = np.moveaxis(x, axis, -1)
    while x.shape[-1] > 1:
        h = x.shape[-1] // 2
        x = x[..., :h] + x[..., h:]
    return x[..., 0]


def tile_partials(c: np.ndarray) -> np.ndarray:
    """(V, ...) per-vertex values -> (tiles, ...) block sums: lanes' halving tree, then the warps'."""
    V = c.shape[0]
    tiles = -(-V // TILE)
    pad = np.zeros((tiles * TILE,) + c.shape[1:])
    pad[:V] = c
    x = pad.reshape((tiles, WARPS, LANES) + c.shape[1:])
    return _halve(_halve(x, 2), 1)


def sum_in_order(parts: np.ndarray) -> np.ndarray:
    """parts (n, ...) summed from 0 in index order."""
    acc = np.zeros(parts.shape[1:])
    for s in range(parts.shape[0]):
        acc = acc + parts[s]
    return acc


# ---- seeds -------------------------------------------------------------------------------------------------------------------
def seeds(rest: np.ndarray, n_bones: int):
    V = len(rest)
    dist = np.zeros(V)
    labels = np.zeros(V, np.int32)
    out = np.zeros(n_bones, np.int32)
    cur = 0
    for b in range(n_bones):
        out[b] = cur
        d = norm2(rest - rest[cur])
        upd = np.ones(V, bool) if b == 0 else d < dist
        dist = np.where(upd, d, dist)
        labels[upd] = b
        cur = int(np.argmax(dist))
    return out, labels, rest[out].copy()


# ---- rigid error -------------------------------------------------------------------------------------------------------------
def rigid_errors(rest: np.ndarray, verts: np.ndarray, xf: np.ndarray) -> np.ndarray:
    """(V, B) e_ij summed over frames in order."""
    T, B = xf.shape[:2]
    e = np.zeros((len(rest), B))
    for t in range(T):
        u = apply_xf(xf[t][None, :, :], rest[:, None, :])
        e = e + norm2(u - verts[t][:, None, :])
    return e


def rigid_error(rest, verts, xf):
    """-> argmin (V), min_error (V), candidates (V, 8) (-1 past B)."""
    e = rigid_errors(rest, verts, xf)
    order = np.argsort(e, axis=1, kind="stable")[:, :N_CAND]
    cand = np.full((len(rest), N_CAND), -1, np.int32)
    cand[:, :order.shape[1]] = order
    return order[:, 0].astype(np.int32), np.take_along_axis(e, order[:, :1], 1)[:, 0], cand


# ---- bone update -------------------------------------------------------------------------------------------------------------
def bone_moments(rest, verts, xf, joints, weights, bone) -> np.ndarray:
    """(T, 16) moments summed over tiles in tile order."""
    T = verts.shape[0]
    a = np.zeros(len(rest))
    for k in range(4):
        hit = (joints[:, k] == bone) & (weights[:, k] > 0)
        a = np.where(hit, weights[:, k], a)
    inf = a > 0
    out = np.zeros((T, 16))
    for t in range(T):
        c = np.zeros((len(rest), 16))
        p = rest[inf]
        q = verts[t][inf] - blend(xf[t], joints[inf], weights[inf], p, bone)
        ai = a[inf]
        a2 = ai * ai
        c[inf, 0] = a2
        for l in range(3):
            c[inf, 1 + l] = a2 * p[:, l]
            c[inf, 4 + l] = ai * q[:, l]
        for l in range(3):
            wp = ai * p[:, l]
            for m in range(3):
                c[inf, 7 + 3 * l + m] = wp * q[:, m]
        out[t] = sum_in_order(tile_partials(c))
    return out


def _jacobi(A: np.ndarray, E: np.ndarray, p: int, q: int) -> None:
    apq = A[:, p, q]
    act = apq != 0
    den = np.where(act, 2.0 * apq, 1.0)
    theta = (A[:, q, q] - A[:, p, p]) / den
    t = np.where(theta >= 0, 1.0, -1.0) / (np.abs(theta) + np.sqrt(theta * theta + 1.0))
    c = 1.0 / np.sqrt(t * t + 1.0)
    s = t * c
    c, s = c[:, None], s[:, None]
    for M, rows in ((A, False), (A, True), (E, False)):
        if rows:
            xp, xq = M[:, p, :].copy(), M[:, q, :].copy()
        else:
            xp, xq = M[:, :, p].copy(), M[:, :, q].copy()
        np_, nq = c * xp - s * xq, s * xp + c * xq
        np_ = np.where(act[:, None], np_, xp)
        nq = np.where(act[:, None], nq, xq)
        if rows:
            M[:, p, :], M[:, q, :] = np_, nq
        else:
            M[:, :, p], M[:, :, q] = np_, nq


def horn_rotation(H: np.ndarray) -> np.ndarray:
    """(n, 3, 3) cross-covariances -> (n, 9) rotations, by Horn's quaternion method with cyclic Jacobi."""
    S = lambda a, b: H[:, a, b]
    n = len(H)
    A = np.zeros((n, 4, 4))
    A[:, 0, 0] = (S(0, 0) + S(1, 1)) + S(2, 2)
    A[:, 0, 1] = S(1, 2) - S(2, 1)
    A[:, 0, 2] = S(2, 0) - S(0, 2)
    A[:, 0, 3] = S(0, 1) - S(1, 0)
    A[:, 1, 1] = (S(0, 0) - S(1, 1)) - S(2, 2)
    A[:, 1, 2] = S(0, 1) + S(1, 0)
    A[:, 1, 3] = S(2, 0) + S(0, 2)
    A[:, 2, 2] = (S(1, 1) - S(0, 0)) - S(2, 2)
    A[:, 2, 3] = S(1, 2) + S(2, 1)
    A[:, 3, 3] = (S(2, 2) - S(0, 0)) - S(1, 1)
    for r in range(4):
        for c in range(r):
            A[:, r, c] = A[:, c, r]
    E = np.tile(np.eye(4), (n, 1, 1))
    with np.errstate(all="ignore"):
        for _ in range(SWEEPS):
            for p, q in PAIRS:
                _jacobi(A, E, p, q)
    best = A[:, 0, 0].copy()
    qv = E[:, :, 0].copy()
    for k in range(1, 4):
        take = A[:, k, k] > best
        best = np.where(take, A[:, k, k], best)
        qv = np.where(take[:, None], E[:, :, k], qv)
    w, x, y, z = qv.T
    nrm = np.sqrt(((w * w + x * x) + y * y) + z * z)
    w, x, y, z = w / nrm, x / nrm, y / nrm, z / nrm
    return np.stack([1.0 - 2.0 * (y * y + z * z), 2.0 * (x * y - w * z), 2.0 * (x * z + w * y),
                     2.0 * (x * y + w * z), 1.0 - 2.0 * (x * x + z * z), 2.0 * (y * z - w * x),
                     2.0 * (x * z - w * y), 2.0 * (y * z + w * x), 1.0 - 2.0 * (x * x + y * y)], -1)


def bone_update(rest, verts, xf, joints, weights, bone, centres):
    """-> (transforms, centres), updated copies."""
    xf, centres = xf.copy(), centres.copy()
    m = bone_moments(rest, verts, xf, joints, weights, bone)
    if not m[0, 0] > 0:
        return xf, centres
    ps = m[:, 1:4] / m[:, :1]
    qs = m[:, 4:7] / m[:, :1]
    H = m[:, 7:16].reshape(-1, 3, 3) - ps[:, :, None] * m[:, None, 4:7]
    R = horn_rotation(H)
    xf[:, bone, :9] = R
    for a in range(3):
        xf[:, bone, 9 + a] = qs[:, a] - ((R[:, 3 * a] * ps[:, 0] + R[:, 3 * a + 1] * ps[:, 1]) + R[:, 3 * a + 2] * ps[:, 2])
    centres[bone] = ps[0]
    return xf, centres


# ---- weight update -----------------------------------------------------------------------------------------------------------
def candidate_lists(joints, weights, cand):
    """-> (c (V, 8) bone ids, -1 past n; n (V,)): used slots in slot order, then new rigid-error candidates in rank order."""
    V = len(joints)
    c = np.full((V, N_CAND), -1, np.int64)
    n = np.zeros(V, np.int64)
    rows = np.arange(V)
    for k in range(4):
        use = weights[:, k] > 0
        c[rows[use], n[use]] = joints[use, k]
        n += use
    for k in range(N_CAND):
        j = cand[:, k].astype(np.int64)
        add = (j >= 0) & (n < N_CAND) & ~(c == j[:, None]).any(1)
        c[rows[add], n[add]] = j[add]
        n += add
    return c, n


def gram(rest, verts, xf, c, n) -> dict:
    """{(a, b): G_ab (V,)} for a <= b: sum_t r_a . r_b, r_a = u_a - v, accumulated where b < n."""
    G = {(a, b): np.zeros(len(rest)) for a in range(N_CAND) for b in range(a, N_CAND)}
    cc = np.maximum(c, 0)
    for t in range(verts.shape[0]):
        r = [apply_xf(xf[t][cc[:, a]], rest) - verts[t] for a in range(N_CAND)]
        for (a, b), g in G.items():
            G[a, b] = np.where(b < n, g + dot3(r[a], r[b]), g)
    return G


def solve_subset(G: dict, idx: tuple):
    """-> (ok (V,), w (V, S), e (V,)) of the KKT solve of subset idx (rule in DESIGN.md §20)."""
    S, M = len(idx), len(idx) + 1
    V = len(G[0, 0])
    g = np.zeros((V, S, S))
    for a in range(S):
        for b in range(a, S):
            g[:, a, b] = g[:, b, a] = G[idx[a], idx[b]]
    s = g[:, 0, 0]
    for a in range(1, S):
        s = np.fmax(s, g[:, a, a])
    ok = s > 0
    A = np.zeros((V, M, M))
    x = np.zeros((V, M))
    with np.errstate(all="ignore"):
        A[:, :S, :S] = g / s[:, None, None]
        A[:, :S, S] = 1.0
        A[:, S, :S] = 1.0
        x[:, S] = 1.0
        det = np.ones(V)
        rows = np.arange(V)
        for k in range(M):
            col = np.abs(A[:, k:, k])
            piv = k + np.argmax(col, 1)
            pv = col.max(1)
            ok &= pv > 0
            tmp = A[rows, piv].copy()
            A[rows, piv] = A[rows, k]
            A[rows, k] = tmp
            tx = x[rows, piv].copy()
            x[rows, piv] = x[rows, k]
            x[rows, k] = tx
            det = det * pv
            for r in range(k + 1, M):
                f = A[:, r, k] / A[:, k, k]
                A[:, r, k + 1:] = A[:, r, k + 1:] - f[:, None] * A[:, k, k + 1:]
                x[:, r] = x[:, r] - f * x[:, k]
        ok &= det > DET_MIN
        for k in range(M - 1, -1, -1):
            acc = x[:, k]
            for c in range(k + 1, M):
                acc = acc - A[:, k, c] * x[:, c]
            x[:, k] = acc / A[:, k, k]
        w = x[:, :S]
        ok &= (w >= 0).all(1)
        e = np.zeros(V)
        for a in range(S):
            gw = np.zeros(V)
            for b in range(S):
                gw = gw + g[:, a, b] * w[:, b]
            e = e + w[:, a] * gw
    return ok, w, e


def weight_update(rest, verts, xf, cand, joints, weights):
    """-> (joints, weights) after one weight update."""
    V = len(rest)
    c, n = candidate_lists(joints, weights, cand)
    G = gram(rest, verts, xf, c, n)
    best_e = G[0, 0].copy()
    best_n = np.ones(V, np.int64)
    best_c = np.zeros((V, 4), np.int64)
    best_w = np.zeros((V, 4))
    best_w[:, 0] = 1.0
    for a in range(1, N_CAND):
        take = (a < n) & (G[a, a] < best_e)
        best_e = np.where(take, G[a, a], best_e)
        best_c[take, 0] = a
    for S in (2, 3, 4):
        for idx in itertools.combinations(range(N_CAND), S):
            ok, w, e = solve_subset(G, idx)
            take = ok & (idx[-1] < n) & (e < best_e)
            best_e = np.where(take, e, best_e)
            best_n[take] = S
            best_c[take, :S] = idx
            best_w[take, :S] = w[take]
    used = (np.arange(4)[None] < best_n[:, None]) & (best_w > 0)
    out_j = np.where(used, np.take_along_axis(c, best_c, 1), 0).astype(np.int32)
    return out_j, np.where(used, best_w, 0.0)


# ---- error -------------------------------------------------------------------------------------------------------------------
def error(rest, verts, xf, joints, weights):
    """-> (frame errors (T + 1): per frame then the sum in frame order, max |v^ - v|^2)."""
    T = verts.shape[0]
    fe = np.zeros(T + 1)
    mx = 0.0
    for t in range(T):
        d2 = norm2(blend(xf[t], joints, weights, rest) - verts[t])
        fe[t] = sum_in_order(tile_partials(d2))
        mx = max(mx, float(d2.max()))
    fe[T] = sum_in_order(fe[:T])
    return fe, mx


# ---- the whole fit -----------------------------------------------------------------------------------------------------------
def fit(vertices, n_bones: int, iterations: int):
    """The whole fit (DESIGN.md §20) -> dict of transforms (T, B, 12), joints, weights, centres, history."""
    verts = np.asarray(vertices, np.float64)
    T, V, _ = verts.shape
    rest = verts[0]
    xf = np.zeros((T, n_bones, 12))
    xf[:, :, [0, 4, 8]] = 1.0
    _, labels, centres = seeds(rest, n_bones)
    joints = np.zeros((V, 4), np.int32)
    weights = np.zeros((V, 4))
    weights[:, 0] = 1.0

    def refit(xf, centres):
        for j in range(n_bones):
            xf, centres = bone_update(rest, verts, xf, joints, weights, j, centres)
        return xf, centres

    for _ in range(CLUSTER_ROUNDS):
        joints[:, 0] = labels
        xf, centres = refit(xf, centres)
        argmin, min_err, _ = rigid_error(rest, verts, xf)
        labels = argmin.copy()
        counts = np.bincount(labels, minlength=n_bones)
        empty = [j for j in range(n_bones) if counts[j] == 0]
        order = sorted(range(V), key=lambda i: (-min_err[i], i))
        for j, i in zip(empty, order):
            labels[i] = j
    joints[:, 0] = labels
    history = [error(rest, verts, xf, joints, weights)[0][T]]
    for _ in range(iterations):
        xf, centres = refit(xf, centres)
        _, _, cand = rigid_error(rest, verts, xf)
        joints, weights = weight_update(rest, verts, xf, cand, joints, weights)
        history.append(error(rest, verts, xf, joints, weights)[0][T])
    return dict(transforms=xf, joints=joints, weights=weights, centres=centres, history=history)
