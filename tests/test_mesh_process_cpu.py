"""Anchor-mesh post-processing without a GPU: properties of the numpy restatement of the decimation (sphere and torus from the
DMC restatement, an open planar grid, the skip rules), the floater rule against scipy's connected components, and the C ABI's
argument validation (no launch)."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp
from scipy.sparse.csgraph import connected_components

import mesh_process_ref as ref
import triposg_vae_ref as tref
from actionmesh_b200.mesh_input import clean_topology


def _dmc_mesh(name):
    field = tref.sphere if name == "sphere" else tref.torus
    v, f = tref.dmc_numpy(tref.dense_grid(field, 97))
    return clean_topology(v.astype(np.float64), f.astype(np.int64))


@pytest.mark.parametrize("name", ["sphere", "torus"])
def test_restatement_decimates_closed_surfaces(name):
    v, f = _dmc_mesh(name)
    assert len(f) > 20000
    _, chi0, vol0 = tref.mesh_stats(v, f)
    v2, f2, rounds = ref.decimate(v, f, 2000)
    assert len(f2) in (1999, 2000) and rounds > 1
    closed, chi, vol = tref.mesh_stats(v2, f2)
    assert closed and chi == chi0 == (2 if name == "sphere" else 0)
    assert abs(vol / vol0 - 1) < 0.01, (vol, vol0)
    assert len(np.unique(f2)) == len(v2)                       # no unreferenced vertex left
    d = ref.point_mesh_distance(v2, v, f)                      # vertices are in voxel units
    assert d.max() <= 0.5, d.max()


def test_restatement_keeps_open_grid_in_plane_and_its_outline():
    v, f = ref.grid_mesh(24)
    v2, f2, _ = ref.decimate(v, f, 200)
    assert len(f2) in (199, 200)
    assert np.all(v2[:, 2] == 0.0)
    assert np.allclose(v2.min(0), v.min(0), rtol=0, atol=1e-12) and np.allclose(v2.max(0), v.max(0), rtol=0, atol=1e-12)
    for corner in ([0, 0], [0, 1], [1, 0], [1, 1]):           # the four corners survive in place
        assert np.min(np.abs(v2[:, :2] - corner).max(1)) <= 1e-12
    # every surviving boundary vertex is still on the outline
    e = np.sort(np.concatenate([f2[:, [0, 1]], f2[:, [1, 2]], f2[:, [2, 0]]]), axis=1)
    u, c = np.unique(e, axis=0, return_counts=True)
    bv = np.unique(u[c == 1])
    on = (np.abs(v2[bv, 0]) < 1e-12) | (np.abs(v2[bv, 0] - 1) < 1e-12) | (np.abs(v2[bv, 1]) < 1e-12) | (np.abs(v2[bv, 1] - 1) < 1e-12)
    assert on.all()


def test_restatement_skip_rules():
    v, f = ref.grid_mesh(6)
    v2, f2, rounds = ref.decimate(v, f, len(f))
    assert rounds == 0 and np.array_equal(v2, v) and np.array_equal(f2, f)
    v3, f3 = ref.remove_floaters(v, f, 0.5)                    # one component: unchanged
    assert v3 is v and f3 is f


def test_postprocessor_skip_rules_need_no_gpu():
    """face_decimation == -1 / <= F and floaters_threshold == 0 run only the host clean (no CUDA call)."""
    from actionmesh_b200.mesh_process import B200MeshPostprocessor

    class M:
        pass

    m = M()
    v, f = ref.grid_mesh(6)
    m.vertices = np.concatenate([v, v[:3]])                   # duplicates that the clean merges, and an unreferenced vertex
    m.vertices = np.concatenate([m.vertices, [[5.0, 5.0, 5.0]]])
    m.faces = np.concatenate([f, f[:2], [[0, 0, 1]]])          # duplicate and degenerate faces
    before = (m.vertices.copy(), m.faces.copy())
    for kw in (dict(face_decimation=-1, floaters_threshold=0.0), dict(face_decimation=len(f), floaters_threshold=0.0),
               dict(face_decimation=10 * len(f))):
        out = B200MeshPostprocessor(device="cpu", **kw).process_mesh(m, seed=1)
        assert np.array_equal(out.vertices, v) and np.array_equal(out.faces, f)
        assert np.asarray(out.vertex_normals).shape == v.shape
    assert np.array_equal(m.vertices, before[0]) and np.array_equal(m.faces, before[1])   # input untouched
    with pytest.raises(Exception):
        B200MeshPostprocessor(device="cpu", face_decimation=10).process_mesh(m)          # no CPU fallback


def test_floater_rule_matches_scipy_components():
    v, f = ref.floater_mesh()
    labels = ref.face_components(f, len(v))
    adj = ref.Adjacency(f, len(v))
    m = adj.nf == 2
    g = sp.coo_matrix((np.ones(m.sum()), (adj.f0[m], adj.f1[m])), shape=(len(f), len(f)))
    n, lab = connected_components(g, directed=False)
    assert n == 6                                              # 2 spheres, 2 triangles, 2 cubes (vertex contact only)
    for c in range(n):                                         # same partition, each labelled by its smallest face
        members = np.flatnonzero(lab == c)
        assert np.all(labels[members] == members.min())
    sizes = np.bincount(lab)
    for thr in (0.02, 0.2, 0.5):
        v2, f2 = ref.remove_floaters(v, f, thr)
        keep = sizes[lab] >= int(sizes.max() * thr)
        assert np.array_equal(f2, np.searchsorted(np.flatnonzero(np.isin(np.arange(len(v)), f[keep])), f[keep]))
        assert np.array_equal(v2, v[np.unique(f[keep])])
    assert len(ref.remove_floaters(v, f, 0.005)[1]) == len(f) - 2         # min 7 faces: only the isolated triangles go
    assert len(ref.remove_floaters(v, f, 0.02)[1]) == len(f) - 2 - 24     # min 29 faces: the 12-face cubes go too
    v3, f3 = ref.remove_floaters(v, f, 2.0)                                 # nothing kept: unchanged
    assert v3 is v and f3 is f


def test_mesh_abi_validation_without_launch(amb_lib):
    from actionmesh_b200 import _lib

    P = 16
    err = lambda: amb_lib.amb_last_error().decode()  # noqa: E731
    assert _lib.ABI_VERSION == amb_lib.amb_abi_version() == 17
    assert amb_lib.amb_mesh_adjacency(None, 4, 4, P, P, P, P, P, None) < 0 and "null pointer" in err()
    assert amb_lib.amb_mesh_adjacency(P, -1, 4, P, P, P, P, P, None) < 0 and "bad mesh size" in err()
    assert amb_lib.amb_mesh_adjacency(P, 1 << 30, 4, P, P, P, P, P, None) < 0 and "bad mesh size" in err()
    assert amb_lib.amb_mesh_edges(P, 4, 4, P, P, P, P, P, P, None, None) < 0 and "null pointer" in err()
    assert amb_lib.amb_mesh_quadrics(P, P, -2, P, P, P, P, None) < 0 and "bad mesh size" in err()
    assert amb_lib.amb_mesh_collapse_select(P, P, P, 4, P, P, P, P, -1, P, P, P, P, P, P, P, None) < 0 and "edge count" in err()
    assert amb_lib.amb_mesh_collapse_apply(P, 4, 4, P, P, P, C.c_uint64(0), P, P, None, None) < 0 and "null pointer" in err()
    assert amb_lib.amb_mesh_compact_faces(P, 4, None, P, None, 0, P, P, None) < 0 and "null pointer" in err()   # labels w/o sizes
    assert amb_lib.amb_mesh_compact_faces(P, 4, None, None, None, 0, P, P, None) < 0 and "alias" in err()
    assert amb_lib.amb_mesh_compact_vertices(P, 4, P, 4, P, P, P, P, None) < 0 and "alias" in err()
    assert amb_lib.amb_mesh_components(None, 4, 4, 1, P, P, None) < 0 and "null pointer" in err()
    assert amb_lib.amb_mesh_component_sizes(P, -1, P, None) < 0 and "bad mesh size" in err()
    # zero-size work is a successful no-op without a launch
    assert amb_lib.amb_mesh_adjacency(P, 0, 4, P, P, P, P, P, None) == 0
    assert amb_lib.amb_mesh_edges(P, 0, 0, P, P, P, P, P, P, P, None) == 0
    assert amb_lib.amb_mesh_quadrics(P, P, 0, P, P, P, P, None) == 0
    assert amb_lib.amb_mesh_collapse_apply(P, 0, 4, P, P, P, C.c_uint64(0), P, P, P, None) == 0
    assert amb_lib.amb_mesh_compact_faces(P, 0, None, None, None, 0, P, 32, None) == 0
    assert amb_lib.amb_mesh_compact_vertices(P, 0, P, 0, P, P, P, 32, None) == 0
    assert amb_lib.amb_mesh_component_sizes(P, 0, P, None) == 0
