"""numpy float64 restatement of csrc/mesh_process.cu: parallel quadric edge-collapse decimation, round by round, and the
floater rule.  Every floating-point operation is an elementwise numpy op (round to nearest, no FMA) in the kernels' order, and
every per-vertex sum runs in the kernels' order, so the CUDA path must reproduce these arrays bit for bit."""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp

DET_REL = 1e-10
BOUNDARY_WEIGHT = 100.0
MIN_COS2 = 0.0625
NO_KEY = np.uint64((1 << 64) - 1)


def cross(a, b):
    return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                     a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], axis=1)


def dot(a, b):
    return (a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]) + a[:, 2] * b[:, 2]


def tri_normal(p0, p1, p2):
    return cross(p1 - p0, p2 - p0)


def plane_terms(u, d, w):
    """(n, 10) terms w * (p_i p_j), p = (u, d), upper triangle row by row."""
    p = [u[:, 0], u[:, 1], u[:, 2], d]
    return np.stack([w * (p[i] * p[j]) for i in range(4) for j in range(i, 4)], axis=1)


def face_plane_terms(p0, n):
    nn = dot(n, n)
    ok = nn > 0
    t = np.zeros((len(n), 10))
    ln = np.sqrt(nn[ok])
    u = n[ok] / ln[:, None]
    t[ok] = plane_terms(u, -dot(u, p0[ok]), 0.5 * ln)
    return t, ok


def boundary_plane_terms(pa, pb, n):
    e = pb - pa
    m = cross(e, n)
    mm = dot(m, m)
    ok = mm > 0
    t = np.zeros((len(n), 10))
    ln = np.sqrt(mm[ok])
    u = m[ok] / ln[:, None]
    t[ok] = plane_terms(u, -dot(u, pa[ok]), BOUNDARY_WEIGHT * dot(e[ok], e[ok]))
    return t, ok


def quadric_error(q, p):
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    r0 = ((q[:, 0] * x + q[:, 1] * y) + q[:, 2] * z) + q[:, 3]
    r1 = ((q[:, 1] * x + q[:, 4] * y) + q[:, 5] * z) + q[:, 6]
    r2 = ((q[:, 2] * x + q[:, 5] * y) + q[:, 7] * z) + q[:, 8]
    r3 = ((q[:, 3] * x + q[:, 6] * y) + q[:, 8] * z) + q[:, 9]
    return ((x * r0 + y * r1) + z * r2) + r3


def f32_round_up(x):
    f = x.astype(np.float32)
    lo = f.astype(np.float64) < x
    f[lo] = np.nextafter(f[lo], np.float32(np.inf))
    return f


# ---- adjacency ---------------------------------------------------------------------------------------------------------------
class Adjacency:
    """vertex -> face CSR (each list in face order), the edges ordered by (a, b) with face count and (up to 2) faces, flags."""

    def __init__(self, faces: np.ndarray, n_vertices: int):
        F = len(faces)
        cv = faces.reshape(-1)
        cf = np.repeat(np.arange(F), 3)
        order = np.lexsort((cf, cv))
        self.deg = np.bincount(cv, minlength=n_vertices)
        self.off = np.concatenate([[0], np.cumsum(self.deg)])
        self.vf = cf[order]
        he = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])
        hf = np.tile(np.arange(F), 3)
        key = he.min(1).astype(np.int64) * n_vertices + he.max(1)
        order = np.lexsort((hf, key))
        ks, fs = key[order], hf[order]
        uniq, start, counts = np.unique(ks, return_index=True, return_counts=True)
        self.a, self.b, self.nf = uniq // n_vertices, uniq % n_vertices, counts
        self.f0 = np.where(counts <= 2, fs[start], -1)
        self.f1 = np.where(counts == 2, fs[np.minimum(start + 1, len(fs) - 1)], -1)
        flags = np.zeros(n_vertices, dtype=np.uint8)
        for m, bit in ((counts == 1, 1), (counts > 2, 2)):
            flags[self.a[m]] |= bit
            flags[self.b[m]] |= bit
        self.flags = flags
        ones = np.ones(len(uniq))
        A = sp.coo_matrix((np.concatenate([ones, ones]), (np.concatenate([self.a, self.b]), np.concatenate([self.b, self.a]))),
                          shape=(n_vertices, n_vertices)).tocsr()
        self.A = A

    def pairs(self, v):
        """(edge-local index, face) for every face of v[i], in face order."""
        d = self.deg[v]
        rep = np.repeat(np.arange(len(v)), d)
        k = np.arange(d.sum()) - np.repeat(np.cumsum(d) - d, d)
        return rep, self.vf[self.off[v][rep] + k]


def _ordered_sum(q, owner, terms, n):
    """q[owner[i]] += terms[i] in the order the terms are given (per owner), vectorised over owners."""
    order = np.argsort(owner, kind="stable")
    owner, terms = owner[order], terms[order]
    cnt = np.bincount(owner, minlength=n)
    first = np.cumsum(cnt) - cnt
    rank = np.arange(len(owner)) - first[owner]
    for k in range(int(rank.max(initial=-1)) + 1):
        s = rank == k
        q[owner[s]] = q[owner[s]] + terms[s]


def quadrics(pos, faces, adj: Adjacency):
    V = len(pos)
    q = np.zeros((V, 10))
    p0, p1, p2 = pos[faces[:, 0]], pos[faces[:, 1]], pos[faces[:, 2]]
    ft, ok = face_plane_terms(p0, tri_normal(p0, p1, p2))
    owner = np.repeat(np.arange(V), adj.deg)
    keep = ok[adj.vf]                                             # the kernel skips zero-area faces
    _ordered_sum(q, owner[keep], ft[adj.vf][keep], V)             # vf is sorted by (vertex, face)
    bnd = np.flatnonzero(adj.nf == 1)
    if len(bnd):
        a, b, f = adj.a[bnd], adj.b[bnd], adj.f0[bnd]
        fp = [pos[faces[f, i]] for i in range(3)]
        bt, ok = boundary_plane_terms(pos[a], pos[b], tri_normal(*fp))
        a, b, bt = a[ok], b[ok], bt[ok]
        owner = np.concatenate([a, b])
        other = np.concatenate([b, a])
        order = np.lexsort((other, owner))
        _ordered_sum(q, owner[order], np.concatenate([bt, bt])[order], V)
    return q


# ---- one round -----------------------------------------------------------------------------------------------------------------
def _faces_stay_valid(pos, faces, adj, v, other, x):
    rep, f = adj.pairs(v)
    fc = faces[f]
    skip = (fc == other[rep][:, None]).any(1)
    old = pos[fc]
    new = old.copy()
    hit = fc == v[rep][:, None]
    new[hit] = np.repeat(x[rep], 3, axis=0).reshape(-1, 3, 3)[hit]
    n_old = tri_normal(old[:, 0], old[:, 1], old[:, 2])
    n_new = tri_normal(new[:, 0], new[:, 1], new[:, 2])
    nn_new, nn_old = dot(n_new, n_new), dot(n_old, n_old)
    d = dot(n_new, n_old)
    bad = ~(nn_new > 0) | ((nn_old > 0) & (~(d > 0) | (d * d < MIN_COS2 * (nn_new * nn_old))))
    out = np.zeros(len(v), dtype=bool)
    np.logical_or.at(out, rep, bad & ~skip)
    return ~out


def select(pos, q, faces, adj: Adjacency):
    """-> (keys (E,) uint64, targets (E, 3), m2 (V,) uint64): key = NO_KEY for invalid collapses."""
    a, b, nf, fl = adj.a, adj.b, adj.nf, adj.flags
    E, V = len(a), len(pos)
    ok = (nf <= 2) & (((fl[a] | fl[b]) & 2) == 0) & ~(((fl[a] & fl[b] & 1) != 0) & (nf != 1))
    common = np.asarray((adj.A @ adj.A)[a, b]).reshape(-1) if E else np.zeros(0)
    ok &= common == nf
    idx = np.flatnonzero(ok)
    ea, eb = a[idx], b[idx]
    qs = q[ea] + q[eb]
    pa, pb = pos[ea], pos[eb]
    pm = (pa + pb) * 0.5
    x = pa.copy()
    cost = quadric_error(qs, pa)
    e_b, e_m = quadric_error(qs, pb), quadric_error(qs, pm)
    s = e_b < cost
    x[s], cost[s] = pb[s], e_b[s]
    s = e_m < cost
    x[s], cost[s] = pm[s], e_m[s]
    Q = [qs[:, i] for i in range(10)]
    c00, c01 = Q[4] * Q[7] - Q[5] * Q[5], Q[2] * Q[5] - Q[1] * Q[7]
    c02, c11 = Q[1] * Q[5] - Q[2] * Q[4], Q[0] * Q[7] - Q[2] * Q[2]
    c12, c22 = Q[1] * Q[2] - Q[0] * Q[5], Q[0] * Q[4] - Q[1] * Q[1]
    det = (Q[0] * c00 + Q[1] * c01) + Q[2] * c02
    solve = np.abs(det) > DET_REL * ((Q[0] * Q[4]) * Q[7])
    with np.errstate(divide="ignore", invalid="ignore"):
        xs = np.stack([-((c00 * Q[3] + c01 * Q[6]) + c02 * Q[8]) / det, -((c01 * Q[3] + c11 * Q[6]) + c12 * Q[8]) / det,
                       -((c02 * Q[3] + c12 * Q[6]) + c22 * Q[8]) / det], axis=1)
        es = quadric_error(qs, xs)
    s = solve & (es <= cost)
    x[s], cost[s] = xs[s], es[s]
    cost = np.where(cost > 0, cost, 0.0)
    good = _faces_stay_valid(pos, faces, adj, ea, eb, x) & _faces_stay_valid(pos, faces, adj, eb, ea, x)
    keys = np.full(E, NO_KEY, dtype=np.uint64)
    targets = np.zeros((E, 3))
    targets[idx] = x
    idx, cost = idx[good], cost[good]
    keys[idx] = (f32_round_up(cost).view(np.uint32).astype(np.uint64) << np.uint64(32)) | idx.astype(np.uint64)
    m1 = np.full(V, NO_KEY, dtype=np.uint64)
    np.minimum.at(m1, a[idx], keys[idx])
    np.minimum.at(m1, b[idx], keys[idx])
    m2 = m1.copy()
    np.minimum.at(m2, a, m1[b])
    np.minimum.at(m2, b, m1[a])
    return keys, targets, m2


def round_limit(win_keys: np.ndarray, win_nf: np.ndarray, n_faces: int, target: int):
    """The key limit of a round and the faces it removes: every winner, unless that passes `target`; then the cheapest winners
    in key order up to the first that reaches it."""
    removed = int(win_nf.sum())
    if n_faces - removed >= target:
        return NO_KEY, removed
    order = np.argsort(win_keys, kind="stable")
    cum = np.cumsum(win_nf[order])
    k = int(np.argmax(n_faces - cum <= target))
    return win_keys[order[k]], int(cum[k])


def drop_unreferenced(pos, faces):
    used = np.zeros(len(pos), dtype=bool)
    used[faces.reshape(-1)] = True
    remap = np.cumsum(used) - 1
    return pos[used], remap[faces]


def one_round(pos, q, faces, target: int, adj: Adjacency | None = None):
    """One decimation round of a mesh with more than `target` faces -> (positions, quadrics, faces) after it, or None when
    no valid collapse is left.  The inputs are not modified; `adj` is Adjacency(faces, len(pos)) when the caller has it."""
    V = len(pos)
    if adj is None:
        adj = Adjacency(faces, V)
    keys, targets, m2 = select(pos, q, faces, adj)
    win = (keys != NO_KEY) & (keys == m2[adj.a]) & (keys == m2[adj.b])
    if not win.any():
        return None
    limit, removed = round_limit(keys[win], adj.nf[win], len(faces), target)
    w = np.flatnonzero(win & (keys <= limit))
    a, b = adj.a[w], adj.b[w]
    remap = np.arange(V)
    remap[b] = a
    pos, q = pos.copy(), q.copy()
    pos[a] = targets[w]
    q[a] = q[a] + q[b]
    faces = remap[faces]
    faces = faces[(faces[:, 0] != faces[:, 1]) & (faces[:, 1] != faces[:, 2]) & (faces[:, 0] != faces[:, 2])]
    return pos, q, faces


def decimate(vertices: np.ndarray, faces: np.ndarray, target: int):
    """-> (vertices (V', 3) float64, faces (F', 3) int64, rounds); the input must be clean (mesh_input.clean_topology)."""
    pos = np.array(vertices, dtype=np.float64)
    faces = np.asarray(faces, dtype=np.int64)
    q = None
    rounds = 0
    while len(faces) > target:
        adj = Adjacency(faces, len(pos))
        if q is None:
            q = quadrics(pos, faces, adj)
        state = one_round(pos, q, faces, target, adj)
        if state is None:
            break
        pos, q, faces = state
        rounds += 1
    pos, faces = drop_unreferenced(pos, faces)
    return pos, faces, rounds


# ---- floaters -------------------------------------------------------------------------------------------------------------------
def face_components(faces: np.ndarray, n_vertices: int) -> np.ndarray:
    """Smallest face index of each face's component; faces are joined through edges held by exactly 2 faces (trimesh's
    face_adjacency).  Min-label propagation with pointer jumping."""
    adj = Adjacency(faces, n_vertices)
    m = adj.nf == 2
    f0, f1 = adj.f0[m], adj.f1[m]
    labels = np.arange(len(faces))
    while True:
        lo = np.minimum(labels[f0], labels[f1])
        new = labels.copy()
        np.minimum.at(new, f0, lo)
        np.minimum.at(new, f1, lo)
        new = new[new]
        if np.array_equal(new, labels):
            return labels
        labels = new


def remove_floaters(vertices: np.ndarray, faces: np.ndarray, threshold: float):
    """The reference's remove_floaters rule with faces and vertices kept in their original order."""
    labels = face_components(faces, len(vertices))
    sizes = np.bincount(labels, minlength=len(faces))
    if np.count_nonzero(sizes) <= 1:
        return vertices, faces
    min_faces = int(sizes.max() * threshold)
    keep = (sizes > 0) & (sizes >= min_faces)
    if not keep.any():
        return vertices, faces
    return drop_unreferenced(vertices, faces[keep[labels]])


# ---- test meshes ----------------------------------------------------------------------------------------------------------------
def grid_mesh(n: int = 24, size: float = 1.0):
    """Open (n x n)-cell planar grid in z = 0, two triangles per cell."""
    a = np.linspace(0.0, size, n + 1)
    x, y = np.meshgrid(a, a, indexing="ij")
    verts = np.stack([x.ravel(), y.ravel(), np.zeros(x.size)], axis=1)
    i, j = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    v00 = (i * (n + 1) + j).ravel()
    v10, v01, v11 = v00 + n + 1, v00 + 1, v00 + n + 2
    faces = np.concatenate([np.stack([v00, v10, v11], 1), np.stack([v00, v11, v01], 1)])
    return verts, faces


def fan_mesh(n: int = 1000):
    """A disk of n triangles around one centre vertex (degree n)."""
    t = np.arange(n) * (2 * np.pi / n)
    verts = np.concatenate([[[0.0, 0.0, 0.0]], np.stack([np.cos(t), np.sin(t), 0.05 * np.sin(3 * t)], 1)])
    k = np.arange(n)
    faces = np.stack([np.zeros(n, dtype=np.int64), 1 + k, 1 + (k + 1) % n], 1)
    return verts, faces


def uv_sphere(center, radius, n_lat, n_lon):
    lat = np.linspace(0, np.pi, n_lat + 1)[1:-1]
    lon = np.linspace(0, 2 * np.pi, n_lon, endpoint=False)
    la, lo = np.meshgrid(lat, lon, indexing="ij")
    ring = np.stack([np.sin(la) * np.cos(lo), np.sin(la) * np.sin(lo), np.cos(la)], -1).reshape(-1, 3)
    verts = np.concatenate([[[0, 0, 1.0]], ring, [[0, 0, -1.0]]]) * radius + np.asarray(center, dtype=np.float64)
    faces = []
    top, bot = 0, len(verts) - 1
    r = lambda i, j: 1 + i * n_lon + j % n_lon  # noqa: E731
    for j in range(n_lon):
        faces.append([top, r(0, j), r(0, j + 1)])
        faces.append([bot, r(n_lat - 2, j + 1), r(n_lat - 2, j)])
    for i in range(n_lat - 2):
        for j in range(n_lon):
            faces.append([r(i, j), r(i + 1, j), r(i + 1, j + 1)])
            faces.append([r(i, j), r(i + 1, j + 1), r(i, j + 1)])
    return verts, np.asarray(faces, dtype=np.int64)


def cube(center, size):
    c = np.array([[x, y, z] for x in (0, 1) for y in (0, 1) for z in (0, 1)], dtype=np.float64) * size + center
    faces = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6], [0, 2, 6],
                      [0, 6, 4], [1, 5, 7], [1, 7, 3]])
    return c, faces


def concat(*meshes):
    vs, fs, n = [], [], 0
    for v, f in meshes:
        vs.append(v)
        fs.append(f + n)
        n += len(v)
    return np.concatenate(vs), np.concatenate(fs)


def floater_mesh():
    """A large sphere, a small sphere, two isolated triangles and two cubes touching only at a vertex, faces interleaved."""
    tri = (np.array([[3.0, 3, 3], [3.1, 3, 3], [3, 3.1, 3]]), np.array([[0, 1, 2]]))
    tri2 = (np.array([[-3.0, 3, 3], [-3.1, 3, 3], [-3, 3.1, 3]]), np.array([[0, 1, 2]]))
    c1 = cube(np.array([2.0, -2, 0]), 0.5)
    c2 = (c1[0] + 0.5, c1[1])                          # shares only the corner (2.5, -1.5, 0.5) geometrically
    v, f = concat(uv_sphere([0, 0, 0], 1.0, 24, 32), tri, uv_sphere([0, 0, 2.5], 0.3, 8, 10), c1, tri2, c2)
    from actionmesh_b200.mesh_input import clean_topology

    v, f = clean_topology(v, f)                        # merges the shared cube corner into one vertex
    perm = np.random.default_rng(0).permutation(len(f))
    return v, f[perm]


def blob_field(n_blobs: int = 40, seed: int = 0):
    """A multi-component test field for triposg_vae_ref.dense_grid: xyz (P, 3) fp32 torch -> (P, 1) logits, positive inside.
    A sum of seeded Gaussian blobs around two cluster centres, which mesh to two large components, plus one small isolated
    blob whose component is far below 2 % of the largest one's faces."""
    import torch

    rng = np.random.default_rng(seed)
    hub = np.where(np.arange(n_blobs)[:, None] % 3 == 2, [0.5, 0.1, 0.0], [-0.5, -0.1, 0.0])
    centres = np.concatenate([hub + rng.uniform(-0.28, 0.28, (n_blobs, 3)), [[0.0, -0.7, 0.7]]])
    radii = np.concatenate([rng.uniform(0.1, 0.2, n_blobs), [0.045]])
    c = torch.from_numpy(centres.astype(np.float32))
    inv = torch.from_numpy((1.0 / (radii * radii)).astype(np.float32))

    def field(xyz):
        cd, invd = c.to(xyz.device), inv.to(xyz.device)
        out = []
        for p in xyz.split(1 << 18):
            d2 = ((p[:, None, :] - cd[None]) ** 2).sum(-1)
            out.append((torch.exp(-d2 * invd).sum(-1, keepdim=True) - 0.5) * 8.0)
        return torch.cat(out)

    return field


def soup_mesh(V: int = 200, F: int = 600, seed: int = 3):
    """A random non-manifold face soup, cleaned."""
    from actionmesh_b200.mesh_input import clean_topology

    rng = np.random.default_rng(seed)
    return clean_topology(rng.standard_normal((V, 3)), rng.integers(0, V, (F, 3)))


def point_mesh_distance(points: np.ndarray, verts: np.ndarray, faces: np.ndarray, k: int = 24) -> np.ndarray:
    """Distance of each point to the triangle mesh (exact point-triangle distance over the k triangles with the nearest
    centroids, so never below the true distance)."""
    from scipy.spatial import cKDTree

    tri = verts[faces]
    _, cand = cKDTree(tri.mean(1)).query(points, k=min(k, len(faces)))
    cand = cand.reshape(len(points), -1)
    best = np.full(len(points), np.inf)
    for j in range(cand.shape[1]):
        t = tri[cand[:, j]]
        best = np.minimum(best, _point_triangle(points, t[:, 0], t[:, 1], t[:, 2]))
    return best


def _point_triangle(p, a, b, c):
    """Vectorised closest-point-on-triangle distance (Ericson, Real-Time Collision Detection 5.1.5)."""
    ab, ac, ap = b - a, c - a, p - a
    d1, d2 = np.einsum("ij,ij->i", ab, ap), np.einsum("ij,ij->i", ac, ap)
    bp, cp = p - b, p - c
    d3, d4 = np.einsum("ij,ij->i", ab, bp), np.einsum("ij,ij->i", ac, bp)
    d5, d6 = np.einsum("ij,ij->i", ab, cp), np.einsum("ij,ij->i", ac, cp)
    va, vb, vc = d3 * d6 - d5 * d4, d5 * d2 - d1 * d6, d1 * d4 - d3 * d2
    with np.errstate(divide="ignore", invalid="ignore"):
        denom = 1.0 / (va + vb + vc)
        v, w = vb * denom, vc * denom
        q = a + ab * v[:, None] + ac * w[:, None]
        cases = [
            ((d1 <= 0) & (d2 <= 0), a),
            ((d3 >= 0) & (d4 <= d3), b),
            ((d6 >= 0) & (d5 <= d6), c),
            ((vc <= 0) & (d1 >= 0) & (d3 <= 0), a + ab * (d1 / (d1 - d3))[:, None]),
            ((vb <= 0) & (d2 >= 0) & (d6 <= 0), a + ac * (d2 / (d2 - d6))[:, None]),
            ((va <= 0) & (d4 - d3 >= 0) & (d5 - d6 >= 0), b + (c - b) * ((d4 - d3) / ((d4 - d3) + (d5 - d6)))[:, None]),
        ]
    done = np.zeros(len(p), dtype=bool)
    for m, pt in cases:
        m = m & ~done
        q[m] = pt[m]
        done |= m
    return np.linalg.norm(p - q, axis=1)
