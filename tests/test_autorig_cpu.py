"""The automatic rig without a GPU (DESIGN.md §22): the topology rules on hand-built pair tables, the numpy restatement on
a synthetic articulated animation, the rigged GLB writer against an independent glTF evaluator, the command line, and
the kernels' register budget."""
from __future__ import annotations

import os
import re
import subprocess

import numpy as np
import pytest

import autorig_ref as ref
import autorig_synthetic as syn
import glb_check
from actionmesh_b200 import autorig, gltf
from test_rig_cpu import evaluate


@pytest.fixture(autouse=True)
def _mat4(monkeypatch):
    monkeypatch.setitem(glb_check.NCOMP, "MAT4", 16)


def _tables(B, adjacent=(), cost=None):
    P = B * (B - 1) // 2
    count = np.zeros(P, np.int32)
    for i, j in adjacent:
        count[autorig.pair_index(min(i, j), max(i, j), B)] = 3
    return count, np.ones(P) if cost is None else np.asarray(cost, np.float64)


# ---- topology --------------------------------------------------------------------------------------------------------------
def test_one_bone_is_one_root_joint():
    bones, parent, pair = autorig.skeleton_topology(np.zeros(0), np.zeros(0), [2.0])
    assert bones.tolist() == [0] and parent.tolist() == [-1] and pair.tolist() == [-1]


def test_root_is_the_heaviest_bone_and_the_order_depth_first():
    # chain 0 - 1 - 2 and 1 - 3 - 4, all adjacent; bone 1 and 3 tie for the largest weight: the lower index wins
    count, cost = _tables(5, [(0, 1), (1, 2), (1, 3), (3, 4)])
    bones, parent, pair = autorig.skeleton_topology(count, cost, [1.0, 5.0, 1.0, 5.0, 1.0])
    assert bones.tolist() == [1, 0, 2, 3, 4]
    assert parent.tolist() == [-1, 0, 0, 0, 3]
    assert pair.tolist() == [-1, autorig.pair_index(0, 1, 5), autorig.pair_index(1, 2, 5), autorig.pair_index(1, 3, 5),
                             autorig.pair_index(3, 4, 5)]
    rb, rp, rq = ref.topology(count, cost, [1.0, 5.0, 1.0, 5.0, 1.0])
    assert np.array_equal(rb, bones) and np.array_equal(rp, parent) and np.array_equal(rq, pair)


def test_adjacent_pairs_come_first_and_ties_go_to_the_lower_pair():
    # a triangle of adjacent pairs with equal costs: (0, 1) and (0, 2) win over (1, 2); a cheaper non-adjacent pair loses
    B = 4
    count, cost = _tables(B, [(0, 1), (0, 2), (1, 2), (2, 3)])
    cost[autorig.pair_index(1, 3, B)] = 0.0
    bones, parent, _ = autorig.skeleton_topology(count, cost, [3.0, 1.0, 1.0, 1.0])
    edges = {frozenset((int(bones[k]), int(bones[parent[k]]))) for k in range(1, B)}
    assert edges == {frozenset((0, 1)), frozenset((0, 2)), frozenset((2, 3))}


def test_disconnected_parts_join_through_the_cheapest_non_adjacent_pair():
    B = 5
    count, cost = _tables(B, [(0, 1), (2, 3), (3, 4)])
    cost[:] = 10.0
    cost[autorig.pair_index(1, 4, B)] = 0.5
    cost[autorig.pair_index(0, 2, B)] = 0.7
    bones, parent, pair = autorig.skeleton_topology(count, cost, [1.0, 1.0, 1.0, 9.0, 1.0])
    edges = {frozenset((int(bones[k]), int(bones[parent[k]]))) for k in range(1, B)}
    assert edges == {frozenset((0, 1)), frozenset((2, 3)), frozenset((3, 4)), frozenset((1, 4))}
    assert bones[0] == 3 and (parent[1:] < np.arange(1, B)).all()
    rb, rp, _ = ref.topology(count, cost, [1.0, 1.0, 1.0, 9.0, 1.0])
    assert np.array_equal(rb, bones) and np.array_equal(rp, parent)


# ---- the restatement on a synthetic skeleton -------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def synthetic():
    rest, faces, W = syn.mesh()
    v, _ = syn.animate(rest, W, T=6)
    return rest, faces, W, v, ref.fit(v, faces, 7, autorig.DEFAULT_ROUNDS, autorig.DEFAULT_SWEEPS)


def _as_fit(r, rest) -> autorig.AutoRigFit:
    T, J = r["rotations"].shape[:2]
    mats = r["rotations"].reshape(T, J, 3, 3)
    return autorig.AutoRigFit(parent=r["parent"], bones=r["bones"], positions=r["positions"],
                              rotations=gltf._quaternions(mats), rotation_matrices=mats,
                              root_translations=r["translations"][:, 0], rest=rest, joints=r["joints"],
                              weights=r["weights"], history=r["history"], rms_error=0.0, max_error=0.0, ssdr_rms_error=0.0)


def test_restatement_recovers_a_synthetic_skeleton(synthetic):
    rest, faces, W, v, r = synthetic
    fit = _as_fit(r, rest)
    diag = np.linalg.norm(rest.max(0) - rest.min(0))
    seg = syn.segment_of_bones(fit, W)
    assert syn.tree_edges(fit, seg) == syn.true_edges()
    assert syn.joint_errors(fit, seg).max() <= 1e-3 * diag
    T, V = v.shape[:2]
    assert np.sqrt(r["history"][-1] / (T * V)) / diag <= syn.RMS_BOUND
    h = r["history"]
    assert all(h[i + 1] <= h[i] * (1 + 1e-12) for i in range(len(h) - 1))
    # posed_vertices (numpy matrix products) poses the fit as the kernels' restatement does, to rounding
    import rig_ref

    want = rig_ref.posed(r["rig"], r["rotations"], r["translations"])
    assert np.abs(autorig.posed_vertices(fit) - want).max() <= 1e-12 * max(1.0, np.abs(want).max())


# ---- the writer ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("multi", [False, True])
def test_writer_shows_the_fit_at_every_key(synthetic, tmp_path, multi):
    rest, faces, _, _, r = synthetic
    fit = _as_fit(r, rest)
    visual = None
    if multi:
        pre, suf = np.maximum.accumulate(faces.max(1)), np.minimum.accumulate(faces.min(1)[::-1])[::-1]
        half = int(np.flatnonzero(pre[:-1] < suf[1:])[0]) + 1           # the horizontal tube's faces come first
        lo = int(pre[half - 1]) + 1
        visual = gltf.GltfMultiVisual(vertex_ranges=np.array([[0, lo], [lo, len(rest) - lo]]),
                                      face_ranges=np.array([[0, half], [half, len(faces) - half]]),
                                      uv=np.zeros((len(rest), 2), np.float32), has_uv=np.array([False, True]),
                                      primitive_material=[None, 0], materials=[{"name": "red"}], textures=[],
                                      samplers=[], images=[], image_bytes=[])
    out = tmp_path / "auto.glb"
    gltf.write_auto_rig_glb(out, fit, faces, visual=visual)
    glb_check.check_glb(out)
    loaded = gltf.load_rig(out)
    assert len(loaded.joint_nodes) == 7
    want = autorig.posed_vertices(fit) @ gltf.ANIMATED_GLB_MAP.T
    assert np.abs(evaluate(out) - rest @ gltf.ANIMATED_GLB_MAP.T).max() <= 2.0 ** -18 * 2
    for k in range(len(want)):
        assert np.abs(evaluate(out, key=k) - want[k]).max() <= 2.0 ** -18 * max(1.0, np.abs(want).max()), k


def test_writer_refusals(synthetic, tmp_path):
    rest, faces, _, _, r = synthetic
    fit = _as_fit(r, rest)
    with pytest.raises(ValueError, match="at least one face"):
        gltf.write_auto_rig_glb(tmp_path / "x.glb", fit, np.zeros((0, 3), np.int64))
    bad = _as_fit(r, rest)
    bad.parent = np.roll(bad.parent, 1)
    with pytest.raises(ValueError, match="depth-first tree"):
        gltf.write_auto_rig_glb(tmp_path / "x.glb", bad, faces)


# ---- arguments -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw,match", [
    (dict(vertices=np.full((2, 4, 3), np.nan)), "non-finite"),
    (dict(vertices=np.zeros((0, 4, 3))), "T >= 1"),
    (dict(faces=np.zeros((0, 3))), "F >= 1"),
    (dict(faces=np.array([[0, 1, 4]])), "outside the 4 vertices"),
    (dict(n_joints=0), r"n_joints must be in \[1, 4\]"),
    (dict(n_joints=5), r"n_joints must be in \[1, 4\]"),
    (dict(rounds=-1), "rounds and sweeps"),
    (dict(sweeps=-1), "rounds and sweeps"),
])
def test_argument_refusals(kw, match):
    args = dict(vertices=np.zeros((2, 4, 3)), faces=np.array([[0, 1, 2], [1, 2, 3]]), n_joints=2)
    args.update(kw)
    with pytest.raises(ValueError, match=match):
        autorig.fit_auto_rig(**args)


# ---- the command line ------------------------------------------------------------------------------------------------------------
def test_cli_flag_parsing():
    from actionmesh_b200 import inference

    assert inference.parse_args(["--input", "x.mp4"]).auto_rig == 0
    assert inference.parse_args(["--input", "x.mp4", "--auto_rig", "12", "--skinning_bones", "3"]).auto_rig == 12
    for bad in ("-1", "257"):
        with pytest.raises(SystemExit):
            inference.parse_args(["--input", "x.mp4", "--auto_rig", bad])


def test_cli_flag_writes_the_auto_rigged_glb(synthetic, tmp_path, monkeypatch):
    from actionmesh_b200 import inference
    from actionmesh_b200.pipeline import Mesh

    rest, faces, _, v, r = synthetic
    seen = {}

    class Pipe:
        device = "cpu"

        def __call__(self, input, seed, **kw):
            return [Mesh(vertices=x, faces=faces) for x in v]

    def fake_fit(vertices, f, n_joints, device=None):
        seen["args"] = (vertices, f, n_joints)
        return _as_fit(r, rest)

    monkeypatch.setattr(inference, "load_frames", lambda *a_, **k: type("F", (), {"frames": []})())
    monkeypatch.setattr(inference.autorig, "fit_auto_rig", fake_fit)
    monkeypatch.setattr(inference.render, "B200MeshVisualizer", lambda **k: type("V", (), {"render": lambda *a_, **k_: None})())
    outs = [tmp_path / "plain", tmp_path / "auto"]
    inference.run_actionmesh(Pipe(), "x", str(outs[0]))
    inference.run_actionmesh(Pipe(), "x", str(outs[1]), auto_rig_joints=7)
    names = sorted(p.name for p in outs[0].iterdir())
    assert sorted(p.name for p in outs[1].iterdir()) == sorted(names + ["auto_rigged_mesh.glb"])
    for name in names:
        assert (outs[0] / name).read_bytes() == (outs[1] / name).read_bytes(), name
    assert np.array_equal(seen["args"][0], v) and np.array_equal(seen["args"][1], faces) and seen["args"][2] == 7


# ---- the kernels compile without spills --------------------------------------------------------------------------------------
def test_autorig_kernels_do_not_spill(tmp_path):
    import __graft_entry__ as ge

    obj = str(tmp_path / "autorig.o")
    res = subprocess.run([ge._nvcc(), *ge.NVCC_FLAGS, "-c", os.path.join(ge.CSRC, "autorig.cu"), "-o", obj],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    entries = re.findall(r"Function properties for (\w+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads", res.stdout + res.stderr)
    assert len(entries) >= 12
    for name, _, stores, loads in entries:
        assert stores == "0" and loads == "0", f"{name} spills {stores} B / loads {loads} B"
