"""Stage 0's geometry kernels element by element (-m gpu): dual marching cubes against an independently derived patch table on
dyadic grids (exact vertex bits) and against its numpy restatement (faces), hand-checked cases, the octree primitives
against a torch restatement of the reference's band at every grid side the depth-9 ladder launches, the count -> scan ->
emit compaction from one tile to ~63 k tiles, refine_octree against the reference's own flash_extract_geometry, and
the DMC kernel at production size.  Outputs are written into views of canary-filled buffers, which must survive."""
import resource
import time

import numpy as np
import pytest
import torch

import geometry_exact as gx
import triposg_vae_ref as ref
from conftest import load_golden

pytestmark = pytest.mark.gpu

TABLE = gx.independent_tables()
MULTI = set(np.nonzero(TABLE[1] > 1)[0].tolist())       # the 92 cases with 2, 3 or 4 patches
U8_CANARY = 0xA5
F32_CANARY = 0x7FC0A5A5                                  # a quiet NaN with a recognisable payload
I32_CANARY = -0x5A5A5A5B                                 # 0xA5A5A5A5
PAD = 4099                                               # canary elements on each side of an output view


def _canary(numel, dtype, shape=None):
    """-> (buffer, contiguous view of `numel` elements starting PAD elements in), the rest of the buffer a canary."""
    if dtype == torch.uint8:
        buf = torch.full((numel + 2 * PAD,), U8_CANARY, dtype=torch.uint8, device="cuda")
    else:
        buf = torch.full((numel + 2 * PAD,), F32_CANARY if dtype == torch.float32 else I32_CANARY, dtype=torch.int32,
                         device="cuda").view(dtype)
    view = buf[PAD:PAD + numel]
    return buf, view.view(shape) if shape is not None else view


def _canary_intact(buf):
    raw = buf.view(torch.uint8) if buf.dtype == torch.uint8 else buf.view(torch.int32)
    want = U8_CANARY if buf.dtype == torch.uint8 else (F32_CANARY if buf.dtype == torch.float32 else I32_CANARY)
    return bool((raw[:PAD] == want).all() and (raw[-PAD:] == want).all())


def _dmc(grid_np):
    """The two calls of ops.dual_marching_cubes with every output in a canary buffer -> numpy cases, vertex offsets,
    vertices and faces (the wrapper returns only the last two)."""
    from actionmesh_b200 import ops

    g = torch.from_numpy(np.ascontiguousarray(grid_np, dtype=np.float32)).cuda()
    n, m3 = g.shape[0], (g.shape[0] - 1) ** 3
    dev = torch.cuda.current_device()
    cb, cases = _canary(m3, torch.uint8)
    vs, fs = ops._scan_scratch(m3, g.device), ops._scan_scratch(n ** 3, g.device)
    common = (ops._ptr(g, torch.float32, "grid", dev), n, ops._ptr(cases, torch.uint8, "cases", dev),
              ops._ptr(vs, torch.int32, "vs", dev), ops._ptr(fs, torch.int32, "fs", dev))
    ops._launch(ops._abi.amb_dmc_count, 9, *common)
    nv, nf = int(vs[-1]), int(fs[-1])
    ob, voff = _canary(m3, torch.int32)
    vb, verts = _canary(3 * max(nv, 1), torch.float32, (max(nv, 1), 3))   # the ABI takes no null output
    fb, faces = _canary(3 * max(nf, 1), torch.int32, (max(nf, 1), 3))
    ops._launch(ops._abi.amb_dmc_emit, 0, *common, ops._ptr(voff, torch.int32, "voff", dev),
                ops._ptr(verts, torch.float32, "verts", dev), ops._ptr(faces, torch.int32, "faces", dev))
    torch.cuda.synchronize()
    assert all(_canary_intact(b) for b in (cb, ob, vb, fb)), "a DMC kernel wrote outside its output"
    verts, faces = verts[:nv], faces[:nf]
    wv, wf = ops.dual_marching_cubes(g)                  # the wrapper returns the same arrays
    assert torch.equal(wv.view(torch.int32), verts.view(torch.int32)) and torch.equal(wf, faces)
    return cases.cpu().numpy(), voff.cpu().numpy(), verts.cpu().numpy(), faces.cpu().numpy()


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.int32)


def _check_cells(grid, label):
    """Cases, vertex counts, vertex offsets and vertex bits of the kernel against dmc_expected (independent table)."""
    exp = gx.dmc_expected(grid, TABLE)
    cases, voff, verts, faces = _dmc(grid)
    case = np.where(exp["valid"], exp["case"], 0)
    assert np.array_equal(cases.astype(np.int64), case)
    counts = np.diff(np.append(voff.astype(np.int64), len(verts)))
    assert np.array_equal(counts, exp["count"]), "vertices per cell != independent patch count"
    assert np.array_equal(voff, exp["offsets"]), "vertex_offsets is not the exclusive scan of the counts"
    assert np.array_equal(_bits(verts), _bits(exp["vertices"])), "vertex bits differ from the dyadic expectation"
    reached = np.unique(case[exp["valid"]])
    multi_cells = int(np.isin(case, list(MULTI)).sum())
    print(f"{label}: {len(reached)} distinct cases, {multi_cells} multi-patch cells, "
          f"{len(set(reached.tolist()) & MULTI)} multi-patch cases, {len(verts)} vertices")
    return exp, cases, voff, verts, faces


# ---- all 256 cases, vertices -----------------------------------------------------------------------------------------
def test_every_case_as_an_isolated_cell(amb_lib):
    grid, where = gx.case_grid()
    exp, cases, voff, verts, faces = _check_cells(grid, "isolated cells")
    assert all(cases[where[c]] == c for c in range(256))
    assert exp["valid"].sum() == 256 and len(faces) == 0    # NaN planes leave no quad


@pytest.mark.parametrize("seed", [11, 12])
def test_every_case_on_random_dyadic_grids(amb_lib, seed):
    grid = gx.dyadic_grid(64, seed)
    exp, *_ = _check_cells(grid, f"dyadic 64^3 seed {seed}")
    per_case = np.bincount(exp["case"], minlength=256)
    assert per_case.min() > 0, np.nonzero(per_case == 0)[0]


# ---- faces -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nan_fraction", [0.0, 0.05])
@pytest.mark.parametrize("seed", [21, 22])
def test_faces_on_random_dyadic_grids(amb_lib, seed, nan_fraction):
    grid = gx.dyadic_grid(64, seed, nan_fraction, outside_border=True)
    exp, cases, voff, verts, faces = _check_cells(grid, f"faces seed {seed} nan {nan_fraction}")
    rv, rf = ref.dmc_numpy(grid)
    assert np.array_equal(_bits(verts), _bits(rv)) and np.array_equal(faces.astype(np.int64), rf)
    assert len(faces) == gx.expected_face_count(grid) > 0
    assert gx.faces_nondegenerate(faces)
    assert gx.vertices_in_cells(verts, exp["cell_of_vertex"], 63)
    if nan_fraction:
        near = gx.invalid_near(grid)[exp["cell_of_vertex"]]
        assert gx.directed_edges_paired(faces, keep=lambda a, b: ~near[a] & ~near[b])
    else:
        assert gx.directed_edges_paired(faces) and gx.signed_volume(verts, faces) > 0
    used = set(np.unique(cases).tolist())
    assert MULTI <= used, sorted(MULTI - used)           # every case with more than one patch occurs


# ---- hand-checked cases ---------------------------------------------------------------------------------------------
# A lone inside point at +1 among -1 neighbours cuts the 3 edges it ends in each of its 8 cells at their midpoints, so per
# axis the vertex is the cell origin + (1/2 + 1 + 1) / 3 in a cell below the point and + (1/2 + 0 + 0) / 3 in a cell above.
BELOW = np.float32(2.5) / np.float32(3)
ABOVE = np.float32(0.5) / np.float32(3)
A, B = np.float32(0) + BELOW, np.float32(1) + ABOVE


def _point_vertex(cell_origin, point):
    return np.array([np.float32(o) + (BELOW if o < p else ABOVE) for o, p in zip(cell_origin, point)], dtype=np.float32)


def test_single_inside_point(amb_lib):
    g = np.full((3, 3, 3), -1.0, dtype=np.float32)
    g[1, 1, 1] = 1.0
    _, voff, v, f = _dmc(g)
    want_v = np.array([[a, b, c] for a in (A, B) for b in (A, B) for c in (A, B)], dtype=np.float32)
    want_f = [[0, 1, 3], [0, 3, 2], [0, 4, 5], [0, 5, 1], [0, 2, 6], [0, 6, 4],
              [4, 6, 7], [4, 7, 5], [2, 3, 7], [2, 7, 6], [1, 5, 7], [1, 7, 3]]
    assert np.array_equal(voff, np.arange(8)) and np.array_equal(_bits(v), _bits(want_v))
    assert f.tolist() == want_f
    normal = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    assert (np.einsum("ij,ij->i", normal, v[f].mean(axis=1) - 1.0) > 0).all()   # every face points away from the point

    _, _, vc, fc = _dmc(-g)                              # the complement: same vertices, every quad reversed
    assert np.array_equal(_bits(vc), _bits(want_v))
    assert fc.tolist() == [[0, 2, 3], [0, 3, 1], [0, 1, 5], [0, 5, 4], [0, 4, 6], [0, 6, 2],
                           [4, 5, 7], [4, 7, 6], [2, 6, 7], [2, 7, 3], [1, 3, 7], [1, 7, 5]]
    assert gx.signed_volume(v, f) > 0 > gx.signed_volume(vc, fc)


@pytest.mark.parametrize("case, second", [(9, (2, 2, 1)), (129, (2, 2, 2))])
def test_two_inside_points_in_one_cell(amb_lib, case, second):
    """Inside points (1,1,1) and `second` share cell (1,1,1) as corners 0 and 3 (case 9, a face diagonal) or 0 and 7
    (case 129, the body diagonal).  That cell has two patches, one per point, and the mesh is two separate closed
    octahedra: each vertex is the vertex a lone point would give, and each face is a lone point's face."""
    first = (1, 1, 1)
    g = np.full((4, 4, 4), -1.0, dtype=np.float32)
    g[first], g[second] = 1.0, 1.0
    cases, voff, v, f = _dmc(g)
    assert cases[(1 * 3 + 1) * 3 + 1] == case and TABLE[1][case] == 2
    cells = [(x, y, z) for x in range(3) for y in range(3) for z in range(3)]
    want = []
    for cell in cells:                                   # cell order, then patch order (smallest edge first)
        pts = [p for p in (first, second) if all(c <= q <= c + 1 for c, q in zip(cell, p))]
        want += [_point_vertex(cell, p) for p in pts]
    assert np.array_equal(_bits(v), _bits(np.array(want)))
    assert len(v) == 16 and len(f) == 24 and gx.directed_edges_paired(f) and gx.faces_nondegenerate(f)
    comp = np.array([0 if np.abs(x - np.array(first)).max() < 0.5 else 1 for x in v])   # each within 1/6 of its point
    assert (comp[f] == comp[f][:, :1]).all()             # no face joins the two points' vertices
    for k, p in enumerate((first, second)):
        fk = f[comp[f[:, 0]] == k]
        assert len(fk) == 12 and gx.directed_edges_paired(fk)
        normal = np.cross(v[fk[:, 1]] - v[fk[:, 0]], v[fk[:, 2]] - v[fk[:, 0]])
        assert (np.einsum("ij,ij->i", normal, v[fk].mean(axis=1) - np.array(p)) > 0).all()


# ---- conventions ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("centre, among_outside, among_inside",
                         [(0.0, 0, 8), (-0.0, 0, 8), (1e-45, 8, 0), (np.inf, 0, 0), (-np.inf, 0, 0), (np.nan, 0, 0)])
def test_zero_is_outside_and_non_finite_corners_invalidate(amb_lib, centre, among_outside, among_inside):
    """A centre point among -1 (outside) or +1 (inside) neighbours: 0 and -0 are outside, the smallest subnormal is
    inside, and +-inf or NaN makes all 8 cells around it invalid (no vertex, no face)."""
    for fill, n_verts in ((-1.0, among_outside), (1.0, among_inside)):
        g = np.full((3, 3, 3), fill, dtype=np.float32)
        g[1, 1, 1] = centre
        cases, _, v, f = _dmc(g)
        assert len(v) == n_verts and len(f) == (12 if n_verts else 0), (fill, len(v), len(f))
        if not np.isfinite(centre):
            assert (cases == 0).all()


def test_side_two_gives_vertices_and_no_faces(amb_lib):
    g = np.array([-1, -3, 0, 1, 3, -1, -3, 1], dtype=np.float32).reshape(2, 2, 2)
    cases, voff, v, f = _dmc(g)
    exp = gx.dmc_expected(g, TABLE)
    assert cases.tolist() == [exp["case"][0]] and len(v) == TABLE[1][exp["case"][0]] > 0 and len(f) == 0
    assert np.array_equal(_bits(v), _bits(exp["vertices"]))


# ---- the octree primitives ------------------------------------------------------------------------------------------
def _input_with_trailer(g):
    """A copy of grid g inside a buffer with n^2 values of alternating sign before and after it: a read one x-plane
    outside the grid sees a neighbour of the wrong sign."""
    n = g.shape[0]
    side = torch.arange(n * n, device="cuda", dtype=torch.float32).remainder(2).mul(14.0).sub(7.0)
    buf = torch.cat([side, g.reshape(-1), side])
    return buf[n * n:n * n + n ** 3].view(n, n, n)


@pytest.mark.parametrize("n", gx.SIDES)
def test_near_surface_band(amb_lib, n):
    from actionmesh_b200 import ops

    g = _input_with_trailer(gx.band_grid(n, "cuda"))
    buf, out = _canary(n ** 3, torch.uint8, (n, n, n))
    ops.octree_near_surface(g, out=out)
    want = gx.near_surface_ref(g)
    assert _canary_intact(buf)
    assert torch.equal(out, want), int((out != want).sum())
    assert 0 < int(want.sum()) < n ** 3 or n <= 3


@pytest.mark.parametrize("n", [2, 3, 12, 13, 16])
def test_near_surface_band_matches_reference_golden(amb_lib, n):
    from actionmesh_b200 import ops

    gold = load_golden("octree_fields.pt")["bands"][n]
    g = gx.band_grid(n, "cuda")
    assert ref.sha256(g) == gold["sha256_grid"]
    assert torch.equal(ops.octree_near_surface(g).cpu(), gold["mask"])


@pytest.mark.parametrize("n", gx.SIDES)
def test_dilate_and_mark_upsampled(amb_lib, n):
    from actionmesh_b200 import ops

    gen = torch.Generator(device="cuda").manual_seed(n)
    for density in (0.0, 0.002, 0.3):
        mask = (torch.rand(n, n, n, device="cuda", generator=gen) < density).to(torch.uint8)
        mask *= torch.randint(1, 256, (n, n, n), device="cuda", dtype=torch.uint8, generator=gen)   # any non-zero marks
        if n > 2:
            mask[-1, -1, -1] = 7                         # the last item and the border
        buf, out = _canary(n ** 3, torch.uint8, (n, n, n))
        ops.octree_dilate(mask, out=out)
        assert _canary_intact(buf) and torch.equal(out, gx.dilate_ref(mask))
        if 2 * n - 1 <= 505:
            buf, fine = _canary((2 * n - 1) ** 3, torch.uint8, (2 * n - 1,) * 3)
            ops.octree_mark_upsampled(mask, out=fine)
            assert _canary_intact(buf) and torch.equal(fine, gx.mark_upsampled_ref(mask))


RES = np.array([2.01 / 504, 2.01 / 252 * 1.1, 0.01234567], dtype=np.float32)   # a distinct resolution per axis
LO = np.array([-1.005, -0.7, 0.3], dtype=np.float32)


def _check_points(mask):
    from actionmesh_b200 import ops

    xyz, idx = ops.octree_points(mask, RES, LO)
    want_xyz, want_idx = gx.points_ref(mask, RES, LO)
    assert torch.equal(idx, want_idx), "index is not torch.nonzero order"
    assert torch.equal(xyz.view(torch.int32), want_xyz.view(torch.int32)), "xyz is not fp32(idx) * res + lo"
    return idx.numel()


@pytest.mark.parametrize("n", gx.SIDES)
def test_octree_points(amb_lib, n):
    from actionmesh_b200 import ops

    mask = ops.octree_dilate(ops.octree_near_surface(gx.band_grid(n, "cuda")))
    _check_points(mask)


@pytest.mark.parametrize("n", gx.SIDES)
def test_grid_fill_replace_scatter(amb_lib, n):
    from actionmesh_b200 import ops

    total = n ** 3
    buf, grid = _canary(total, torch.float32, (n, n, n))
    ops.grid_fill(grid, gx.INVALID)
    torch.cuda.synchronize()
    assert _canary_intact(buf) and bool((grid == gx.INVALID).all())
    gen = torch.Generator(device="cuda").manual_seed(n + 1)
    idx = torch.randperm(total, device="cuda", generator=gen)[:max(1, total // 3)].to(torch.int32)
    wide = torch.randn(idx.numel(), 5, device="cuda", generator=gen)
    wide[::7, 2] = gx.INVALID                            # some scattered values are the filler itself
    values = wide[:, 2:]                                 # row stride 5, column 0 at an offset
    ops.grid_scatter(values, idx, grid)
    want = torch.full((total,), gx.INVALID, device="cuda")
    want[idx.long()] = wide[:, 2]
    torch.cuda.synchronize()
    assert _canary_intact(buf) and torch.equal(grid.reshape(-1).view(torch.int32), want.view(torch.int32))
    ops.grid_replace(grid, gx.INVALID, float("nan"))
    want = torch.where(want == gx.INVALID, float("nan"), want)
    torch.cuda.synchronize()
    assert _canary_intact(buf) and torch.equal(grid.reshape(-1).view(torch.int32), want.view(torch.int32))


# ---- the scan, through octree_points (pure compaction) --------------------------------------------------------------
@pytest.mark.parametrize("n", gx.SCAN_SIDES)
def test_scan_tile_offsets(amb_lib, n):
    """The count pass alone: the scratch must hold the exclusive scan of the 2048-item tile counts and then the grand
    total, which the wrapper reads back to size its outputs (checked here before anything is emitted)."""
    from actionmesh_b200 import ops

    gen = torch.Generator(device="cuda").manual_seed(5 * n)
    mask = (torch.rand(n, n, n, device="cuda", generator=gen) < 0.3).to(torch.uint8)
    scratch = ops._scan_scratch(n ** 3, mask.device)
    dev = torch.cuda.current_device()
    ops._launch(ops._abi.amb_octree_count_points, 4, ops._ptr(mask, torch.uint8, "mask", dev), n,
                ops._ptr(scratch, torch.int32, "scratch", dev))
    flat = mask.reshape(-1).int()
    tiles = torch.nn.functional.pad(flat, (0, (-flat.numel()) % 2048)).view(-1, 2048).sum(1)
    want = torch.cat([torch.zeros(1, dtype=torch.int64, device="cuda"), tiles.cumsum(0)]).int()
    assert scratch.numel() == tiles.numel() + 1 and torch.equal(scratch, want)


@pytest.mark.parametrize("n", gx.SCAN_SIDES)
@pytest.mark.parametrize("pattern", ["zeros", "ones", "last", "sparse", "dense"])
def test_scan_compaction(amb_lib, n, pattern):
    gen = torch.Generator(device="cuda").manual_seed(3 * n)
    if pattern in ("zeros", "last"):
        mask = torch.zeros(n, n, n, dtype=torch.uint8, device="cuda")
        if pattern == "last":
            mask[-1, -1, -1] = 1
    elif pattern == "ones":
        mask = torch.ones(n, n, n, dtype=torch.uint8, device="cuda")
    else:
        mask = (torch.rand(n, n, n, device="cuda", generator=gen) < (0.001 if pattern == "sparse" else 0.6)).to(torch.uint8)
    count = _check_points(mask)
    assert count == {"zeros": 0, "ones": n ** 3, "last": 1}.get(pattern, count)


# ---- refine_octree against the reference's flash_extract_geometry ----------------------------------------------------
@pytest.mark.parametrize("name, depth", [("border", 8), ("level", 8), ("thin", 8), ("border", 9), ("level", 9), ("thin", 9)])
def test_refine_octree_matches_reference_golden(amb_lib, name, depth):
    from actionmesh_b200.triposg_vae import refine_octree

    gold = load_golden("octree_fields.pt")["fields"][(name, depth)]
    grid = refine_octree(getattr(gx, name + "_field"), ref.BOUNDS, depth).reshape(-1)
    assert grid.shape[0] == gold["side"] ** 3
    idx = torch.nonzero(torch.isfinite(grid)).reshape(-1).to(torch.int32)
    val = grid[idx.long()]
    assert idx.numel() == gold["count"]
    assert torch.equal(idx[:2000].cpu(), gold["head_index"]) and torch.equal(val[:2000].cpu(), gold["head_values"])
    assert ref.sha256(idx) == gold["sha256_index"] and ref.sha256(val) == gold["sha256_values"]


# ---- production size ------------------------------------------------------------------------------------------------
def test_dmc_at_production_size(amb_lib):
    from actionmesh_b200.triposg_vae import refine_octree

    grid = refine_octree(gx.rippled_field, ref.BOUNDS, 9)
    assert grid.shape == (505, 505, 505)
    g = grid.cpu().numpy()
    cases, voff, v, f = _dmc(g)
    case, valid = gx.cell_cases(g)
    multi_cells = int((np.isin(case, list(MULTI)) & valid).sum())
    assert multi_cells > 0, "the band holds no multi-patch cell"
    t0, r0 = time.time(), resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
    rv, rf = ref.dmc_numpy(g)
    t_np = time.time() - t0
    assert np.array_equal(_bits(v), _bits(rv)) and np.array_equal(f.astype(np.int64), rf)
    assert len(f) == gx.expected_face_count(g) and gx.faces_nondegenerate(f)
    cell_of_vertex = np.repeat(np.arange(504 ** 3), np.diff(np.append(voff.astype(np.int64), len(v))))
    assert gx.vertices_in_cells(v, cell_of_vertex, 504)
    e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]).astype(np.int64), axis=1)
    _, per_edge = np.unique(e[:, 0] * len(v) + e[:, 1], return_counts=True)
    print(f"production 505^3: {len(v)} vertices, {len(f)} faces, {multi_cells} multi-patch cells, "
          f"{len(set(np.unique(case[valid]).tolist()) & MULTI)} multi-patch cases, "
          f"{int((per_edge == 4).sum())} edges with 4 faces, dmc_numpy {t_np:.1f} s, "
          f"host peak RSS {max(r0, resource.getrusage(resource.RUSAGE_SELF).ru_maxrss) / 2 ** 20:.1f} GiB, "
          f"device peak {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")
