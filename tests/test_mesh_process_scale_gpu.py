"""Mesh post-processing on the GPU at the sizes Stage 0 produces (-m gpu), bit for bit against tests/mesh_process_ref.py.

- Kernel by kernel on the depth-9 sphere and torus (over 800 000 faces) and a multi-component blob mesh of about 435 000 faces:
  adjacency, initial quadrics, collapse selection and one applied round.
- Round replay: the whole GPU decimation of those meshes to 40 000 faces, with its first, a middle and its final (key-limited)
  round restated from the GPU's own input state.
- Whole runs of a blob mesh of about 150 000 faces, decimated to 40 000 faces and cleared of floaters below 2 %, through the
  module functions and B200MeshPostprocessor.
- Face components on a 200 000-face strip whose face order runs against it or is shuffled, so that the union needs many
  passes, on 10 000 isolated faces and on the decimated blob mesh."""
from functools import lru_cache

import numpy as np
import pytest
import torch

import mesh_process_ref as ref
import triposg_vae_ref as tref
from actionmesh_b200.mesh_input import clean_topology

pytestmark = pytest.mark.gpu

TARGET = 40000


@lru_cache(maxsize=None)
def _mesh(name):
    """Clean (vertices float64, faces int64) meshes: the depth-9 sphere and torus as the octree decoder meshes them, and the
    seeded blob field meshed on dense grids of 369^3 (about 435 000 faces) and 217^3 (about 150 000 faces)."""
    from actionmesh_b200 import ops
    from actionmesh_b200.triposg_vae import mesh_from_grid, refine_octree

    if name in ("sphere", "torus"):
        field = tref.sphere if name == "sphere" else tref.torus
        v, f = mesh_from_grid(refine_octree(field, tref.BOUNDS, 9), tref.BOUNDS, 9)
    else:
        n = {"blob": 369, "blob_small": 217}[name]
        a = torch.linspace(-1.0, 1.0, n, device="cuda")
        xyz = torch.stack(torch.meshgrid(a, a, a, indexing="ij"), -1).reshape(-1, 3)
        grid = ref.blob_field()(xyz).reshape(n, n, n).contiguous()
        vt, ft = ops.dual_marching_cubes(grid)
        v, f = vt.cpu().numpy(), ft.cpu().numpy()
    return clean_topology(v.astype(np.float64), f.astype(np.int64))


def _same(a, b):
    """Bit-identical float64 arrays (and equal shapes)."""
    return a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64))


def _cuda(v, f):
    return (torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64)).cuda(),
            torch.from_numpy(np.ascontiguousarray(f, dtype=np.int32)).cuda())


@pytest.mark.parametrize("name", ["sphere", "torus", "blob"])
def test_kernels_match_restatement_on_full_size_meshes(amb_lib, name):
    from actionmesh_b200 import ops

    v, f = _mesh(name)
    V, F = len(v), len(f)
    assert F > (800_000 if name != "blob" else 400_000)
    pos, ft = _cuda(v, f)
    work, scan = ops.mesh_scan_scratch(V, F, "cuda")
    adj = ops.mesh_adjacency(ft, V, work, scan)
    off, vf, _, edges, flags = (t.cpu().numpy() for t in adj)
    r = ref.Adjacency(f, V)
    assert np.array_equal(off, r.off) and np.array_equal(vf, r.vf)
    assert np.array_equal(edges, np.stack([r.a, r.b, r.nf, r.f0, r.f1], 1))
    assert np.array_equal(flags, r.flags)

    q = ops.mesh_quadrics(pos, ft, adj)
    rq = ref.quadrics(v, f, r)
    assert _same(q.cpu().numpy(), rq)

    sel = ops.mesh_collapse_select(pos, q, ft, adj)
    keys, targets, m2 = ref.select(v, rq, f, r)
    valid = keys != ref.NO_KEY
    m1 = np.full(V, ref.NO_KEY, dtype=np.uint64)
    np.minimum.at(m1, r.a[valid], keys[valid])
    np.minimum.at(m1, r.b[valid], keys[valid])
    assert np.array_equal(sel["keys"].cpu().numpy().view(np.uint64), keys)
    assert _same(sel["targets"].cpu().numpy(), targets)
    vmin = sel["vertex_min"].cpu().numpy().view(np.uint64)
    assert np.array_equal(vmin[:V], m1) and np.array_equal(vmin[V:], m2)
    win = valid & (keys == m2[r.a]) & (keys == m2[r.b])
    got = sel["winners"].cpu().numpy()
    got = got[np.argsort(got[:, 0].view(np.uint64))]
    assert np.array_equal(got[:, 0].view(np.uint64), np.sort(keys[win]))
    assert np.array_equal(got[:, 1], r.nf[win][np.argsort(keys[win])])
    assert sel["removed"] == int(r.nf[win].sum()) and F - sel["removed"] >= TARGET

    remap = ops.mesh_collapse_apply(adj[3], sel, ops.NO_KEY, pos, q)
    ft = ops.mesh_compact_faces(ft, scan, remap=remap)
    rp, rq, rf = ref.one_round(v, rq, f, TARGET, r)
    assert np.array_equal(ft.cpu().numpy(), rf)
    assert _same(pos.cpu().numpy(), rp) and _same(q.cpu().numpy(), rq)


def _gpu_rounds(v, f, target, capture=()):
    """mesh_process.decimate's loop through ops -> (rounds, {round: ((pos, q, faces) before, (pos, q, faces) after, key-limited)})
    for the rounds in `capture`, as numpy arrays."""
    from actionmesh_b200 import ops
    from actionmesh_b200.mesh_process import _round_limit

    pos, ft = _cuda(v, f)
    V, F = len(v), len(f)
    work, scan = ops.mesh_scan_scratch(V, F, "cuda")
    state = lambda: (pos.cpu().numpy(), q.cpu().numpy(), ft.cpu().numpy().astype(np.int64))  # noqa: E731
    q, rounds, seen = None, 0, {}
    while F > target:
        adj = ops.mesh_adjacency(ft, V, work, scan)
        if q is None:
            q = ops.mesh_quadrics(pos, ft, adj)
        sel = ops.mesh_collapse_select(pos, q, ft, adj)
        if not len(sel["winners"]):
            break
        limit, removed = ops.NO_KEY, sel["removed"]
        if F - removed < target:
            limit, removed = _round_limit(sel["winners"].cpu().numpy(), F, target)
        before = state() if rounds in capture else None
        remap = ops.mesh_collapse_apply(adj[3], sel, limit, pos, q)
        ft = ops.mesh_compact_faces(ft, scan, remap=remap)
        assert ft.shape[0] == F - removed
        F = ft.shape[0]
        if before is not None:
            seen[rounds] = (before, state(), limit != ops.NO_KEY)
        rounds += 1
    return rounds, seen


@pytest.mark.parametrize("name", ["sphere", "torus", "blob"])
def test_round_replay_on_full_size_meshes(amb_lib, name):
    v, f = _mesh(name)
    rounds, _ = _gpu_rounds(v, f, TARGET)
    picks = (0, rounds // 2, rounds - 1)
    again, seen = _gpu_rounds(v, f, TARGET, picks)
    assert again == rounds and sorted(seen) == sorted(set(picks))
    assert seen[rounds - 1][2], "the final round should stop at the target by key"
    for k in sorted(seen):
        (p, q, fc), (gp, gq, gf), _ = seen[k]
        rp, rq, rf = ref.one_round(p, q, fc, TARGET)
        assert np.array_equal(gf, rf), k
        assert _same(gp, rp) and _same(gq, rq), k
    assert len(seen[rounds - 1][1][2]) in (TARGET - 1, TARGET)
    print(f"{name}: {len(f)} faces, {rounds} rounds")


@lru_cache(maxsize=None)
def _blob_small_reference():
    v, f = _mesh("blob_small")
    dv, df, rounds = ref.decimate(v, f, TARGET)
    return (dv, df, rounds), ref.remove_floaters(dv, df, 0.02)


def test_whole_run_matches_restatement(amb_lib):
    from actionmesh_b200 import ops
    from actionmesh_b200.mesh_process import B200MeshPostprocessor, decimate, make_mesh, remove_floaters

    v, f = _mesh("blob_small")
    (dv, df, rounds), (kv, kf) = _blob_small_reference()
    sizes = np.bincount(ref.face_components(df, len(dv)))
    sizes = sizes[sizes > 0]
    assert len(sizes) >= 3 and sizes.min() < int(sizes.max() * 0.02), sizes     # at least one floater to remove
    assert len(kf) < len(df)

    pos, ft = _cuda(v, f)
    work, scan = ops.mesh_scan_scratch(len(v), len(f), "cuda")
    pos, ft, grounds = decimate(pos, ft, TARGET, work, scan)
    assert grounds == rounds
    assert np.array_equal(ft.cpu().numpy(), df) and _same(pos.cpu().numpy(), dv)
    pos, ft = remove_floaters(pos, ft, 0.02, work, scan)
    assert np.array_equal(ft.cpu().numpy(), kf) and _same(pos.cpu().numpy(), kv)

    out = B200MeshPostprocessor(face_decimation=TARGET, floaters_threshold=0.02, verbose=False).process_mesh(make_mesh(v, f))
    assert np.array_equal(np.asarray(out.faces), kf) and _same(np.asarray(out.vertices, dtype=np.float64), kv)
    print(f"blob_small: {len(f)} faces, {rounds} rounds, {len(df)} after decimation, components {sorted(sizes.tolist())}")


def _gpu_components(faces, n_vertices):
    from actionmesh_b200 import ops

    ft = torch.from_numpy(np.ascontiguousarray(faces, dtype=np.int32)).cuda()
    work, scan = ops.mesh_scan_scratch(n_vertices, len(faces), "cuda")
    adj = ops.mesh_adjacency(ft, n_vertices, work, scan)
    labels, sizes = ops.mesh_face_components(adj[3], len(faces))
    return labels.cpu().numpy(), sizes.cpu().numpy()


def _strip(n_quads=100_000):
    """A triangle strip of 2 n_quads faces over two rows of vertices, face i sharing an edge with face i + 1."""
    top, bot, i = np.arange(n_quads + 1), np.arange(n_quads + 1) + n_quads + 1, np.arange(n_quads)
    f = np.stack([np.stack([top[i], bot[i], bot[i + 1]], 1), np.stack([top[i], bot[i + 1], top[i + 1]], 1)], 1)
    return f.reshape(-1, 3), 2 * n_quads + 2


@pytest.mark.parametrize("order", ["reversed", "shuffled"])
def test_components_of_a_long_strip(amb_lib, order):
    f, V = _strip()
    f = f[::-1] if order == "reversed" else f[np.random.default_rng(5).permutation(len(f))]
    labels, sizes = _gpu_components(f, V)
    # one component: every label is face 0 (the restatement's label propagation needs ~one pass per face on the shuffled
    # strip, so the expected labels are written down instead)
    assert np.array_equal(labels, np.zeros(len(f), np.int32))
    assert sizes[0] == len(f) and not sizes[1:].any()
    if order == "reversed":
        assert np.array_equal(labels, ref.face_components(f, V))


def test_components_of_isolated_faces(amb_lib):
    f = np.random.default_rng(2).permutation(30_000).reshape(-1, 3)
    labels, sizes = _gpu_components(f, 30_000)
    want = ref.face_components(f, 30_000)
    assert np.array_equal(labels, want) and np.array_equal(want, np.arange(10_000))
    assert np.array_equal(sizes, np.bincount(want, minlength=len(f)))


def test_components_of_the_decimated_blob_mesh(amb_lib):
    (dv, df, _), _ = _blob_small_reference()
    labels, sizes = _gpu_components(df, len(dv))
    want = ref.face_components(df, len(dv))
    assert np.array_equal(labels, want)
    assert np.array_equal(sizes, np.bincount(want, minlength=len(df)))
