"""A synthetic articulated animation with a known skeleton, for the automatic-rig tests.

Two tubes: a horizontal one along x (segments left2, left1, root, right1, right2) and a vertical one below the root
(segments down1, down2) that shares no face with the first.  Each segment turns about its pivot with a ball joint (a
rotation of up to 60 degrees about a different random axis in every frame), the root also moves, and the vertices follow
by linear blend skinning: one-hot weights, except the ring at each pivot of the horizontal tube, which is split 50 / 50.
"""
from __future__ import annotations

import numpy as np

# segment: (parent, pivot)
SEGMENTS = {
    "root": (None, (0.0, 0.0, 0.0)),
    "left1": ("root", (-0.5, 0.0, 0.0)),
    "left2": ("left1", (-1.0, 0.0, 0.0)),
    "right1": ("root", (0.5, 0.0, 0.0)),
    "right2": ("right1", (1.0, 0.0, 0.0)),
    "down1": ("root", (0.0, -0.2, 0.0)),
    "down2": ("down1", (0.0, -0.7, 0.0)),
}
NAMES = list(SEGMENTS)


def axis_angle(axis, ang) -> np.ndarray:
    a = np.asarray(axis, np.float64)
    a = a / np.linalg.norm(a)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * (K @ K)


def _tube(axis: int, lo: float, hi: float, step: float, radius: float, around: int, offset):
    """Rings of `around` vertices every `step` along `axis` from lo to hi, quads split into two triangles."""
    n_rings = int(round((hi - lo) / step)) + 1
    s = lo + step * np.arange(n_rings)
    ang = 2 * np.pi * np.arange(around) / around
    u, w = radius * np.cos(ang), radius * np.sin(ang)
    others = [k for k in range(3) if k != axis]
    v = np.zeros((n_rings, around, 3))
    v[..., axis] = s[:, None]
    v[..., others[0]] = u[None]
    v[..., others[1]] = w[None]
    v = v.reshape(-1, 3) + np.asarray(offset, np.float64)
    faces = []
    for r in range(n_rings - 1):
        for k in range(around):
            a, b = r * around + k, r * around + (k + 1) % around
            c, d = a + around, b + around
            faces += [[a, b, d], [a, d, c]]
    return v, np.asarray(faces, np.int64), s


def mesh(step: float = 0.05, around: int = 10):
    """-> (rest (V, 3), faces (F, 3), weights (V, 7)) with segment columns in NAMES order."""
    vh, fh, sh = _tube(0, -1.5, 1.5, step, 0.12, around, (0.0, 0.0, 0.0))
    vv, fv, sv = _tube(1, -1.2, -0.25, step, 0.1, around, (0.0, 0.0, 0.0))
    rest = np.concatenate([vh, vv])
    faces = np.concatenate([fh, fv + len(vh)])
    W = np.zeros((len(rest), len(NAMES)))
    col = {n: i for i, n in enumerate(NAMES)}
    x = vh[:, 0]
    for i, xi in enumerate(x):
        if abs(xi) < 0.5 - 1e-9:
            W[i, col["root"]] = 1
        elif abs(abs(xi) - 0.5) <= 1e-9:
            side = "left1" if xi < 0 else "right1"
            W[i, col["root"]], W[i, col[side]] = 0.5, 0.5
        elif abs(xi) < 1.0 - 1e-9:
            W[i, col["left1" if xi < 0 else "right1"]] = 1
        elif abs(abs(xi) - 1.0) <= 1e-9:
            W[i, col["left1" if xi < 0 else "right1"]], W[i, col["left2" if xi < 0 else "right2"]] = 0.5, 0.5
        else:
            W[i, col["left2" if xi < 0 else "right2"]] = 1
    y = vv[:, 1]
    W[len(vh):, col["down1"]] = y > -0.7
    W[len(vh):, col["down2"]] = y <= -0.7
    return rest, faces, W


def animate(rest, W, T: int = 6, seed: int = 0, max_deg: float = 60.0):
    """-> (vertices (T, V, 3), world (T, 7, 3, 4)): frame 0 is the rest pose."""
    rng = np.random.default_rng(seed)
    world = np.zeros((T, len(NAMES), 3, 4))
    for t in range(T):
        for k, name in enumerate(NAMES):
            parent, pivot = SEGMENTS[name]
            q = np.asarray(pivot)
            R = np.eye(3) if t == 0 else axis_angle(rng.standard_normal(3), np.deg2rad(rng.uniform(10, max_deg)))
            local = np.concatenate([R, (q - R @ q)[:, None]], 1)          # rotation about the pivot
            if parent is None:
                if t:
                    local[:, 3] += 0.3 * rng.standard_normal(3)
                world[t, k] = local
            else:
                P = world[t, NAMES.index(parent)]
                world[t, k] = np.concatenate([P[:, :3] @ local[:, :3], (P[:, :3] @ local[:, 3] + P[:, 3])[:, None]], 1)
    u = np.einsum("tkij,vj->tvki", world[..., :3], rest) + world[:, None, :, :, 3]
    return np.einsum("vk,tvki->tvi", W, u), world


def true_edges():
    return {frozenset((NAMES.index(n), NAMES.index(p))) for n, (p, _) in SEGMENTS.items() if p is not None}


# Measured with the restatement at the defaults (4 rounds of 10 sweeps): RMS 1.39e-5 of the diagonal.  The joints stay
# where the SSDR bones put them (within 1.3e-4 of the diagonal of the true pivots, the 50 / 50 rings being what SSDR fits
# least well), and that offset times the joints' rotation is what remains.  More frames do not lower it (1.31e-5 with 12
# or 20 frames), and other random motions end between 1.14e-5 and 1.52e-5 (DESIGN.md §22).
RMS_BOUND = 2e-5


def segment_of_bones(fit, W) -> np.ndarray:
    """The true segment of each joint: the segment most of its dominant vertices follow."""
    dom = np.where(fit.weights.max(1) > 0, fit.joints[np.arange(len(fit.joints)), np.argmax(fit.weights, 1)], -1)
    return np.array([np.bincount(np.argmax(W[dom == k], 1), minlength=len(NAMES)).argmax() for k in range(len(fit.parent))])


def tree_edges(fit, seg) -> set:
    return {frozenset((int(seg[k]), int(seg[fit.parent[k]]))) for k in range(1, len(fit.parent))}


def joint_errors(fit, seg) -> np.ndarray:
    """|c_k - q| for every child joint, q the true pivot between its segment and its parent's."""
    out = []
    for k in range(1, len(fit.parent)):
        a, b = NAMES[seg[k]], NAMES[seg[fit.parent[k]]]
        q = SEGMENTS[a][1] if SEGMENTS[a][0] == b else SEGMENTS[b][1]
        out.append(np.linalg.norm(fit.positions[k] - np.asarray(q)))
    return np.asarray(out)
