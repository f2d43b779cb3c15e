"""Exact expectations for Stage 0's geometry kernels (csrc/geometry.cu, csrc/scan.cuh); not collected by pytest.

  header_tables       the patch table of csrc/dmc_table.cuh, read from the header text.
  independent_tables  the same table derived a second way, from corner components (no code shared with
                      tools/gen_dmc_table.py): see its docstring.
  dyadic_grid         random grids of {-3, -1, 0, +1, +3}: every crossing t = v0 / (v0 - v1) is one of {-0, 1/4, 1/2, 3/4, 1}
                      and every patch sum is exact, so the only rounded operations of a vertex are `s / cnt` and `+ x`.
  dmc_expected        per-cell cases, patch counts, vertex offsets and vertex bits of such a grid, from a table alone.
  case_grid           every one of the 256 cases as an isolated cell, cells separated by NaN planes.
  near_surface_ref    torch restatement of the reference's near-surface band (extract_near_surface_volume_fn + |v| < 0.95).
  dilate_ref, mark_upsampled_ref, points_ref
                      the 3^3 dilation, the upsampled marks and the point compaction of flash_extract_geometry.
  band_grid           deterministic adversarial grids for the band: structure at the border, exact zeros, +-0.95f and its
                      neighbours, -9000, -8999.999 and -10000.
  directed_edges_paired, faces_nondegenerate, vertices_in_cells, signed_volume, expected_face_count
                      mesh invariants that need no patch table.
  border_field, level_field, thin_field, rippled_field
                      analytic logit fields (positive inside) for the octree goldens and the production-size run.
"""
from __future__ import annotations

import os
import re

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "actionmesh_b200", "csrc", "dmc_table.cuh")

# Grid sides the octree and scan tests run: tiny and odd sides, one / two / exactly two scan tiles (2048 items), and the
# depth-9 ladder of refine_octree (coarse grids 64, 127, 253 and their fine masks 127, 253, 505).
SIDES = (2, 3, 12, 13, 16, 64, 127, 253, 505)
SCAN_SIDES = (12, 13, 16, 81, 505)   # 1, 2, exactly 2, 259.5 (past the 256-tile loop of scan_tiles_kernel), ~63 k tiles

CORNERS = [(c & 1, (c >> 1) & 1, (c >> 2) & 1) for c in range(8)]


# ---- the patch table ---------------------------------------------------------------------------------------------------
def header_tables(path: str = HEADER):
    """-> (patch_of_edge (256, 12) int, patch_count (256,) int) parsed from the text of csrc/dmc_table.cuh."""
    text = open(path).read()
    rows = re.findall(r"\{([-\d,\s]+)\},\s*//\s*(\d+)", text)
    assert [int(c) for _, c in rows] == list(range(256)), "kDmcPatchOfEdge must list cases 0..255 in order"
    pe = np.array([[int(v) for v in r.split(",")] for r, _ in rows])
    body = re.search(r"kDmcPatchCount\[256\]\s*=\s*\{([^}]*)\}", text).group(1)
    cnt = np.array([int(v) for v in body.replace(",", " ").split()])
    assert pe.shape == (256, 12) and cnt.shape == (256,)
    return pe, cnt


def edge_ends(e: int):
    """-> (axis, corner at the low end, corner at the high end) of cube edge e."""
    axis, u, v = e >> 2, e & 1, (e >> 1) & 1
    o0, o1 = (i for i in range(3) if i != axis)
    off = [0, 0, 0]
    off[o0], off[o1] = u, v
    c0 = off[0] | (off[1] << 1) | (off[2] << 2)
    return axis, c0, c0 | (1 << axis)


def independent_tables():
    """The patch table derived from corner components, without tools/gen_dmc_table.py:
      * inside corners are joined by cube edges whose two ends are both inside;
      * outside corners are joined by cube edges and by face diagonals, so on an ambiguous face the outside corners
        connect and the inside corners stay separated;
      * a crossing edge belongs to the patch named by (component of its inside end, component of its outside end): on the
        surface of a cube that pair names exactly one contour loop;
      * patches are numbered by their smallest edge index.
    -> (patch_of_edge (256, 12) with -1 for no crossing, patch_count (256,))."""
    pairs = [(a, b) for a in range(8) for b in range(a + 1, 8)]
    dist = {(a, b): sum(x != y for x, y in zip(CORNERS[a], CORNERS[b])) for a, b in pairs}
    pe, cnt = np.full((256, 12), -1), np.zeros(256, dtype=np.int64)
    for case in range(256):
        ins = [(case >> k) & 1 for k in range(8)]
        comp = list(range(8))

        def root(x):
            while comp[x] != x:
                x = comp[x]
            return x

        for a, b in pairs:
            if ins[a] == ins[b] and (dist[a, b] == 1 or (dist[a, b] == 2 and not ins[a])):
                comp[root(a)] = root(b)
        keys = {}
        for e in range(12):
            _, a, b = edge_ends(e)
            if ins[a] != ins[b]:
                key = (root(a), root(b)) if ins[a] else (root(b), root(a))
                pe[case, e] = keys.setdefault(key, len(keys))
        cnt[case] = len(keys)
    return pe, cnt


# ---- DMC grids and expectations ----------------------------------------------------------------------------------------
DYADIC = np.array([-3.0, -1.0, 0.0, 1.0, 3.0], dtype=np.float32)


def dyadic_grid(n: int, seed: int, nan_fraction: float = 0.0, outside_border: bool = False) -> np.ndarray:
    """(n, n, n) fp32 grid of values drawn from {-3, -1, 0, +1, +3}, optionally with NaN points and an all-outside border."""
    rng = np.random.default_rng(seed)
    g = DYADIC[rng.integers(0, len(DYADIC), (n, n, n))]
    if nan_fraction:
        g[rng.random((n, n, n)) < nan_fraction] = np.nan
    if outside_border:
        outside = DYADIC[rng.integers(0, 3, (n, n, n))]
        for axis in range(3):
            for side in (0, n - 1):
                sl = [slice(None)] * 3
                sl[axis] = side
                g[tuple(sl)] = outside[tuple(sl)]
    return g


def cell_corners(g: np.ndarray):
    """The 8 corner views of the (n-1)^3 cells, corner c at offset (c & 1, (c >> 1) & 1, (c >> 2) & 1)."""
    m = g.shape[0] - 1
    return [g[dx:dx + m, dy:dy + m, dz:dz + m] for dx, dy, dz in CORNERS]


def cell_cases(g: np.ndarray):
    """-> (case (m,m,m) int64 with bit c set when corner c > 0, valid (m,m,m): all 8 corners finite)."""
    corners = cell_corners(g)
    case = np.zeros(corners[0].shape, dtype=np.int64)
    valid = np.ones(corners[0].shape, dtype=bool)
    for k, c in enumerate(corners):
        case |= (c > 0).astype(np.int64) << k
        valid &= np.isfinite(c)
    return case, valid


def dmc_expected(g: np.ndarray, tables=None):
    """Vertices of a dyadic grid from a patch table alone (default: independent_tables).

    Each patch sum s is accumulated exactly in float64 (every t is a multiple of 1/4) and checked to be exact in fp32; the
    vertex is then fp32(s) / fp32(cnt) and + fp32(cell origin), each rounded once in fp32 as the kernel does.
    -> dict(case, valid, count (m^3,), offsets (m^3,) int64, vertices (V, 3) fp32, cell_of_vertex (V,))."""
    pe, npatch = independent_tables() if tables is None else tables
    g = np.ascontiguousarray(g, dtype=np.float32)
    m = g.shape[0] - 1
    case, valid = cell_cases(g)
    case = np.where(valid, case, 0).reshape(-1)
    count = npatch[case]
    offsets = np.cumsum(count) - count
    nv = int(count.sum())
    s = np.zeros((nv, 3))
    cnt = np.zeros(nv)
    corners = [c.reshape(-1).astype(np.float64) for c in cell_corners(g)]
    for e in range(12):
        axis, c0, c1 = edge_ends(e)
        o0, o1 = (i for i in range(3) if i != axis)
        p = pe[case, e]
        sel = p >= 0
        vid = offsets[sel] + p[sel]
        a, b = corners[c0][sel], corners[c1][sel]
        t = a / (a - b)
        assert np.isin(t, [0.0, 0.25, 0.5, 0.75, 1.0]).all(), "not a dyadic grid"
        s[vid, axis] += t
        s[vid, o0] += (e & 1)
        s[vid, o1] += (e >> 1) & 1
        cnt[vid] += 1
    assert (cnt >= 3).all() and np.array_equal(s.astype(np.float32).astype(np.float64), s)
    cell_of_vertex = np.repeat(np.arange(m ** 3), count)
    origin = np.stack(np.unravel_index(cell_of_vertex, (m, m, m)), axis=-1).astype(np.float32)
    verts = (s.astype(np.float32) / cnt.astype(np.float32)[:, None]).astype(np.float32) + origin
    return dict(case=case, valid=valid.reshape(-1), count=count, offsets=offsets, vertices=verts.astype(np.float32),
                cell_of_vertex=cell_of_vertex)


def case_grid():
    """A grid in which every case 0..255 is one isolated cell: cell k sits at corner block (3i, 3j, 3k) of a 7^3 lattice
    and every third grid plane is NaN, so no other cell is valid.  Inside corners take +1 or +3, outside ones -3, -1 or 0,
    cycling with the cell, so crossings land on 1/4, 1/2, 3/4 and 1.  -> (grid (21, 21, 21) fp32, {case: cell index})."""
    k, n = 7, 21
    g = np.full((n, n, n), np.nan, dtype=np.float32)
    where = {}
    m = n - 1
    for case in range(256):
        i, j, l = case // (k * k), (case // k) % k, case % k
        for c, (dx, dy, dz) in enumerate(CORNERS):
            r = case * 8 + c
            v = (1.0, 3.0)[r % 2] if (case >> c) & 1 else (-3.0, -1.0, 0.0)[r % 3]
            g[3 * i + dx, 3 * j + dy, 3 * l + dz] = v
        where[case] = (3 * i * m + 3 * j) * m + 3 * l
    return g, where


# ---- table-free mesh invariants ----------------------------------------------------------------------------------------
def directed_edges_paired(faces: np.ndarray, keep=None) -> bool:
    """Every directed edge a -> b occurs as often as its reverse b -> a: consistently wound quads around every grid edge.
    `keep(a, b)` (bool arrays) restricts the check to some edges."""
    f = np.asarray(faces, dtype=np.int64)
    a = np.concatenate([f[:, 0], f[:, 1], f[:, 2]])
    b = np.concatenate([f[:, 1], f[:, 2], f[:, 0]])
    if keep is not None:
        sel = keep(a, b)
        a, b = a[sel], b[sel]
    base = int(max(a.max(initial=0), b.max(initial=0))) + 1
    fwd = np.sort(a * base + b)
    rev = np.sort(b * base + a)
    return bool(np.array_equal(fwd, rev))


def faces_nondegenerate(faces: np.ndarray) -> bool:
    """No face repeats a vertex: the 4 vertices of a quad lie in 4 different cells."""
    f = np.asarray(faces)
    return bool(((f[:, 0] != f[:, 1]) & (f[:, 1] != f[:, 2]) & (f[:, 2] != f[:, 0])).all())


def vertices_in_cells(verts: np.ndarray, cell_of_vertex: np.ndarray, m: int) -> bool:
    """Every vertex lies in its cell's closed unit box: it is a mean of crossings on the cell's edges."""
    origin = np.stack(np.unravel_index(cell_of_vertex, (m, m, m)), axis=-1)
    return bool(((verts >= origin) & (verts <= origin + 1)).all())


def signed_volume(verts: np.ndarray, faces: np.ndarray) -> float:
    """Volume enclosed by the faces (float64), positive when they are wound outward from the inside (logit > 0) region."""
    v = verts.astype(np.float64)
    f = np.asarray(faces, dtype=np.int64)
    return float(np.einsum("ij,ij->i", v[f[:, 0]], np.cross(v[f[:, 1]], v[f[:, 2]])).sum() / 6.0)


def expected_face_count(g: np.ndarray) -> int:
    """2 x the grid edges whose ends are finite and on different sides of 0 and whose 4 surrounding cells exist and have 8
    finite corners, counted straight from the grid."""
    n = g.shape[0]
    fin = np.isfinite(g)
    _, valid = cell_cases(g)
    total = 0
    for axis in range(3):
        lo = [slice(None)] * 3
        hi = [slice(None)] * 3
        lo[axis], hi[axis] = slice(0, n - 1), slice(1, n)
        a, b = g[tuple(lo)], g[tuple(hi)]
        cross = fin[tuple(lo)] & fin[tuple(hi)] & ((a > 0) != (b > 0))
        # the 4 cells around edge p -> p + e_axis are p - {0, 1} along the two other axes: all must exist and be valid
        vb = np.moveaxis(valid, axis, 0)
        around = vb[:, 1:, 1:] & vb[:, :-1, 1:] & vb[:, 1:, :-1] & vb[:, :-1, :-1]
        c = np.moveaxis(cross, axis, 0)[:, 1:n - 1, 1:n - 1]
        total += int((c & around).sum())
    return 2 * total


def invalid_near(g: np.ndarray) -> np.ndarray:
    """(m^3,) bool: cells within one cell (26-neighbourhood) of a cell with a non-finite corner."""
    _, valid = cell_cases(g)
    bad = torch.from_numpy(~valid)[None, None].float()
    return (F.max_pool3d(bad, 3, 1, 1)[0, 0] > 0).numpy().reshape(-1)


# ---- the octree primitives ---------------------------------------------------------------------------------------------
INVALID = -10000.0
F095 = np.float32(0.95)
SPECIAL = np.array([0.0, -0.0, F095, -F095, np.nextafter(F095, 0), np.nextafter(F095, 2), np.nextafter(-F095, 0),
                    np.nextafter(-F095, -2), -9000.0, -8999.999, INVALID, np.nextafter(np.float32(-9000), 0), 1e-45,
                    -1e-45, 0.5, -0.5], dtype=np.float32)


def band_grid(n: int, device="cpu") -> torch.Tensor:
    """Deterministic adversarial (n, n, n) fp32 grid for the near-surface band (integer hashing, no RNG): a slanted plane
    of +2 / -3 that cuts the border, unqueried (-10000) points, and a third of the points replaced by SPECIAL values."""
    i = torch.arange(n, dtype=torch.int64, device=device)
    x, y, z = i.view(-1, 1, 1), i.view(1, -1, 1), i.view(1, 1, -1)
    h = ((x * 73856093) ^ (y * 19349663) ^ (z * 83492791)) & 0xFFFFFF
    g = torch.where((x + 2 * y - z) * 4 > 2 * n, 2.0, -3.0).to(torch.float32).expand(n, n, n)
    g = torch.where(h % 7 == 0, INVALID, g)
    special = torch.from_numpy(SPECIAL).to(device)
    return torch.where(h % 3 == 0, special[(h >> 5) % len(SPECIAL)], g).contiguous()


def near_surface_ref(g: torch.Tensor) -> torch.Tensor:
    """The reference's band, restated: a point is marked when it is valid (v > -9000) and torch.sign of one of its 6 face
    neighbours differs from its own, or when |v| < 0.95 (compared in fp32).  Neighbours come from replicate padding, and
    a neighbour <= -9000 (or NaN) is replaced by the point itself.  -> uint8 (n, n, n)."""
    p = F.pad(g[None, None], (1, 1, 1, 1, 1, 1), mode="replicate")[0, 0]
    n = g.shape[0]
    s = torch.sign(g)
    differs = torch.zeros_like(g, dtype=torch.bool)
    for axis in range(3):
        for d in (0, 2):
            sl = [slice(1, n + 1)] * 3
            sl[axis] = slice(d, d + n)
            nb = p[tuple(sl)]
            nb = torch.where(nb > -9000.0, nb, g)
            differs |= torch.sign(nb) != s
    thr = torch.tensor(0.95, dtype=torch.float32, device=g.device)
    return ((differs & (g > -9000.0)) | (g.abs() < thr)).to(torch.uint8)


def dilate_ref(mask: torch.Tensor) -> torch.Tensor:
    """3^3 dilation with zero padding (the reference's ones-Conv3d(3, padding=1) followed by > 0) -> uint8 0 / 1."""
    return (F.max_pool3d((mask != 0).float()[None, None], 3, 1, 1)[0, 0] > 0).to(torch.uint8)


def mark_upsampled_ref(mask: torch.Tensor) -> torch.Tensor:
    """(n,n,n) -> (2n-1)^3 uint8: fine[2x, 2y, 2z] = (mask[x, y, z] != 0), zeros elsewhere."""
    n = mask.shape[0]
    fine = torch.zeros((2 * n - 1,) * 3, dtype=torch.uint8, device=mask.device)
    fine[::2, ::2, ::2] = (mask != 0).to(torch.uint8)
    return fine


def points_ref(mask: torch.Tensor, resolution, bbox_min):
    """torch.where(mask > 0) in grid order -> (xyz = fp32(idx) * resolution then + bbox_min, each op rounded on its own,
    linear index int32)."""
    n = mask.shape[0]
    idx = torch.nonzero(mask.reshape(-1)).reshape(-1)
    ijk = torch.stack([idx // (n * n), (idx // n) % n, idx % n], dim=1).float()
    res = torch.tensor(np.asarray(resolution, dtype=np.float32), device=mask.device)
    lo = torch.tensor(np.asarray(bbox_min, dtype=np.float32), device=mask.device)
    prod = ijk * res
    return prod + lo, idx.to(torch.int32)


# ---- analytic fields: xyz (P, 3) fp32 -> (P, 1) fp32 logits, positive inside ----------------------------------------------
def border_field(xyz):
    """A ball of radius 1.1 centred at (0.25, 0, 0): it leaves the +-1.005 box, so the band reaches the grid border."""
    x, y, z = xyz[:, 0:1] - 0.25, xyz[:, 1:2], xyz[:, 2:3]
    return (1.21 - (x * x + y * y + z * z)) * 32.0


def grid_coordinate(i: int, r: int, lo: float = -1.005, hi: float = 1.005) -> float:
    """fp32(i) * fp32(size / r) + fp32(lo), as the points of every octree level after the first are computed."""
    step = np.float32((hi - lo) / r)
    return float(np.float32(np.float32(i) * step) + np.float32(lo))


def level_field(xyz, r: int = 252):
    """A ball with exact zeros and +-0.95f at grid points of the octree levels after the first (the grid coordinates of
    level r are those of level 2r at even indices): inside the ball the logit is +0 (x > 0) or -0 (x <= 0) on the plane
    z = z0, exactly +0.95f on the plane y = y1 and exactly -0.95f on the plane y = y2."""
    x, y, z = xyz[:, 0:1], xyz[:, 1:2], xyz[:, 2:3]
    z0, y1, y2 = grid_coordinate(r // 2 + 2, r), grid_coordinate(r // 2 - 8, r), grid_coordinate(r // 2 + 11, r)
    ball = (0.5 - (x * x + y * y + z * z)) * 16.0
    dz = z - z0
    inside = ball > 0
    v = torch.where((dz == 0) & inside, torch.where(x > 0, dz * ball, -(dz * ball)), ball)
    v = torch.where((y == y1) & inside, torch.full_like(v, 0.95), v)
    return torch.where((y == y2) & inside, torch.full_like(v, -0.95), v)


def thin_field(xyz):
    """Several components and features thinner than a cell of the first level (2.01 / 63 = 0.032): two balls, a disc
    about 0.02 thick whose logit stays below 0.95, and three small balls of radius 0.02, united with max."""
    x, y, z = xyz[:, 0:1], xyz[:, 1:2], xyz[:, 2:3]

    def ball(cx, cy, cz, r, k):
        dx, dy, dz = x - cx, y - cy, z - cz
        return (r * r - (dx * dx + dy * dy + dz * dz)) * k

    v = torch.maximum(ball(-0.45, 0.0, 0.0, 0.3, 32.0), ball(0.45, 0.1, 0.0, 0.25, 32.0))
    slab = (0.005 - (y - 0.6) * (y - 0.6) * 40.0) * 64.0 - (x * x + z * z) * 8.0
    v = torch.maximum(v, slab)
    for c in ((0.0, -0.6, 0.3), (0.7, -0.5, -0.5), (-0.3, 0.5, -0.7)):
        v = torch.maximum(v, ball(*c, 0.02, 4096.0))
    return v


def rippled_field(xyz):
    """A ball of radius 0.6 with a sin-product ripple of period ~3 cells of the final depth-9 grid: the ripple folds the
    surface within a cell, so the band holds cells with two, three or four patches."""
    x, y, z = xyz[:, 0:1], xyz[:, 1:2], xyz[:, 2:3]
    k = 520.0
    return (0.36 - (x * x + y * y + z * z)) * 64.0 + torch.sin(x * k) * torch.sin(y * k) * torch.sin(z * k) * 0.6
