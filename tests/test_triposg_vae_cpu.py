"""Stage 0's anchor-mesh path without a GPU: the fp32 decode restatement against the reference's own TripoSG VAE, the numpy
dual-marching-cubes restatement on analytic surfaces, the committed patch table (also against an independent derivation),
the octree resolution ladder and the grid sides the geometry tests run, and the torch restatement of the near-surface band
against the reference's own band."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import geometry_exact as gx
import triposg_vae_ref as ref
from conftest import ROOT, load_golden


def test_fp32_decode_restatement_matches_reference():
    g = load_golden("triposg_vae_tiny.pt")
    c = g["config"]
    sd = ref.make_state_dict(c["width_decoder"], c["num_attention_heads"], c["num_layers_decoder"], seed=g["seed"])
    out = ref.decode_fp32(sd, g["z"], g["points"], c["num_attention_heads"], c["num_layers_decoder"])
    err = float((out - g["logits"]).norm() / g["logits"].norm())
    assert out.shape == g["logits"].shape == (1, 4096, 1) and err <= 1e-5, err


@pytest.mark.parametrize("name", ["sphere", "torus"])
def test_dmc_restatement_on_analytic_surfaces(name):
    n = 97
    field = ref.sphere if name == "sphere" else ref.torus
    grid = ref.dense_grid(field, n)
    verts, faces = ref.dmc_numpy(grid)
    voxel = 2.0 / (n - 1)
    v = verts * voxel - 1.0
    closed, chi, vol = ref.mesh_stats(v, faces)
    assert closed, "every edge must be shared by exactly two faces"
    assert chi == (2 if name == "sphere" else 0), chi
    exact = 4 / 3 * math.pi * ref.SPHERE_R ** 3 if name == "sphere" else 2 * math.pi ** 2 * ref.TORUS_R * ref.TORUS_r ** 2
    assert vol > 0 and abs(vol / exact - 1) < 0.01, (vol, exact)
    dist = ref.sphere_distance(v) if name == "sphere" else ref.torus_distance(v)
    assert dist.max() <= 0.5 * voxel, dist.max() / voxel
    assert len(np.unique(faces)) == len(verts)          # no cell of a NaN-free grid emits an unused vertex


def test_dmc_restatement_drops_quads_next_to_nan_cells():
    grid = ref.dense_grid(ref.sphere, 49)
    cut = grid.copy()
    cut[30:, :, :] = np.nan                 # the +x cap is not finite: its cells and their quads disappear
    v_all, f_all = ref.dmc_numpy(grid)
    v_cut, f_cut = ref.dmc_numpy(cut)
    assert 0 < len(f_cut) < len(f_all)
    assert v_cut[np.unique(f_cut)][:, 0].max() <= 29.0
    closed, _, _ = ref.mesh_stats(v_cut, f_cut)
    assert not closed                        # an open boundary where the quads were dropped


def test_patch_table_header_is_generated():
    res = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "gen_dmc_table.py"), "--check"], capture_output=True,
                         text=True)
    assert res.returncode == 0, res.stdout + res.stderr


def test_patch_table_properties():
    pe, npatch = (np.array(t) for t in ref.dmc_tables())
    assert npatch[0] == npatch[255] == 0 and npatch[1] == 1
    for case in range(256):
        used = pe[case][pe[case] >= 0]
        assert set(used.tolist()) == set(range(npatch[case]))
        assert all(len(np.nonzero(pe[case] == p)[0]) >= 3 for p in range(npatch[case]))   # a patch has >= 3 crossings
    # two inside corners on a face diagonal stay separated (corners 0 and 3 of the z = 0 face)
    assert npatch[0b00001001] == 2


def test_patch_table_header_matches_independent_derivation():
    """csrc/dmc_table.cuh, read as text, equals the table derived from corner components (geometry_exact)."""
    pe, cnt = gx.header_tables()
    ipe, icnt = gx.independent_tables()
    assert np.array_equal(pe, ipe) and np.array_equal(cnt, icnt)
    assert np.bincount(cnt).tolist() == [2, 162, 82, 8, 2]


def test_dyadic_expectation_matches_restatement():
    """On a dyadic grid the vertex bits from the independent table equal dmc_numpy's, and its mesh has the table-free
    invariants the GPU tests assert."""
    g = gx.dyadic_grid(24, 5, outside_border=True)
    exp = gx.dmc_expected(g)
    v, f = ref.dmc_numpy(g)
    assert np.array_equal(exp["vertices"].view(np.int32), v.view(np.int32))
    assert len(f) == gx.expected_face_count(g) > 0 and gx.faces_nondegenerate(f) and gx.directed_edges_paired(f)
    assert gx.vertices_in_cells(v, exp["cell_of_vertex"], 23) and gx.signed_volume(v, f) > 0


def test_geometry_sides_cover_the_depth9_ladder():
    """Every grid the depth-9 refinement launches a geometry kernel on is a side the exact tests run: each level's grid
    n = r + 1 and each fine mask 2n - 1 that mark_upsampled writes."""
    from actionmesh_b200.triposg_vae import octree_resolutions

    sides = [r + 1 for r in octree_resolutions(9)]
    fine = [2 * n - 1 for n in sides[:-1]]
    assert set(sides) | set(fine) <= set(gx.SIDES), sorted((set(sides) | set(fine)) - set(gx.SIDES))
    assert fine[-1] == sides[-1] == max(gx.SIDES) and max(gx.SCAN_SIDES) == sides[-1]


@pytest.mark.parametrize("n", [2, 3, 12, 13, 16])
def test_band_restatement_matches_reference(n):
    """geometry_exact.near_surface_ref equals the reference's extract_near_surface_volume_fn + |v| < 0.95 (golden) on the
    adversarial band grids."""
    gold = load_golden("octree_fields.pt")["bands"][n]
    g = gx.band_grid(n)
    assert ref.sha256(g) == gold["sha256_grid"]
    assert torch.equal(gx.near_surface_ref(g), gold["mask"])


def test_octree_resolution_ladder():
    from actionmesh_b200.triposg_vae import octree_resolutions

    assert octree_resolutions(9) == [63, 126, 252, 504]
    assert octree_resolutions(8) == [63, 126, 252]
    assert octree_resolutions(7) == [63, 126]


def test_state_dict_keys_match_reference():
    """The decoder-side keys B200TripoSGVAE.load_state_dict reads are exactly the ones the golden's reference model took."""
    keys = set(ref.make_state_dict(256, 2, 2))
    assert {k.split(".")[0] for k in keys} == {"post_quant", "decoder"}
    assert "decoder.blocks.2.attn2.norm_cross.weight" in keys and "decoder.blocks.0.attn1.to_q.weight" in keys
    assert torch.load(os.path.join(ROOT, "tests", "golden", "triposg_vae_tiny.pt"), weights_only=False)["config"]["num_layers_decoder"] == 2
