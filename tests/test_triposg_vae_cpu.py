"""Stage 0's anchor-mesh path without a GPU: the fp32 decode restatement against the reference's own TripoSG VAE, the numpy
dual-marching-cubes restatement on analytic surfaces, the committed patch table and the octree resolution ladder."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

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
