"""The automatic rig on the GPU (DESIGN.md §22): every kernel of csrc/autorig.cu bit for bit against autorig_ref, at small
and production sizes, the whole fit against the restatement, the synthetic skeleton, and a run on the tiny checkpoint
tree."""
from __future__ import annotations

import numpy as np
import pytest
import torch

import autorig_ref as ref
import autorig_synthetic as syn
import glb_check
from actionmesh_b200 import autorig, ops
from actionmesh_b200 import rig as rigmod
from test_rig_cpu import evaluate

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _mat4(monkeypatch):
    monkeypatch.setitem(glb_check.NCOMP, "MAT4", 16)


def _same(a, b) -> bool:
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype == np.float64:
        return a.shape == b.shape and np.array_equal(a.view(np.uint64), np.asarray(b, np.float64).view(np.uint64))
    return a.shape == b.shape and np.array_equal(a, b)


def _cuda(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def grid_mesh(V: int, seed: int = 0):
    """A wavy sheet of about V vertices: (rest (V, 3), faces (F, 3) int32)."""
    n = int(np.ceil(np.sqrt(V)))
    x, y = np.meshgrid(np.linspace(0, 1, n), np.linspace(0, 1, n))
    rest = np.stack([x.ravel(), y.ravel(), 0.1 * np.sin(7 * x.ravel()) * np.cos(5 * y.ravel())], -1)[:V]
    idx = np.arange(n * n).reshape(n, n)
    a, b, c, d = idx[:-1, :-1].ravel(), idx[:-1, 1:].ravel(), idx[1:, :-1].ravel(), idx[1:, 1:].ravel()
    faces = np.concatenate([np.stack([a, b, d], -1), np.stack([a, d, c], -1)])
    faces = faces[(faces < V).all(1)]
    return rest, np.ascontiguousarray(faces, dtype=np.int32)


def random_skin(rest, B, seed=0):
    """joints / weights (V, 4) in skin_weight_update's layout: 1 to 4 used slots, some unused ones in between, ties."""
    rng = np.random.default_rng(seed)
    V = len(rest)
    region = np.minimum((rest[:, 0] * B).astype(np.int64), B - 1)        # spatially coherent dominant bones
    joints = np.stack([region] + [rng.integers(0, B, V) for _ in range(3)], 1).astype(np.int32)
    weights = rng.choice([0.0, 0.125, 0.25, 0.5], size=(V, 4))
    weights[:, 0] = np.where(rng.random(V) < 0.5, 1.0, 0.5)
    joints = np.where(weights > 0, joints, 0).astype(np.int32)
    return joints, weights


def random_transforms(T, B, seed=0):
    rng = np.random.default_rng(seed)
    xf = np.zeros((T, B, 12))
    for t in range(T):
        for b in range(B):
            q = rng.standard_normal(4)
            q /= np.linalg.norm(q)
            x, y, z, w = q
            xf[t, b, :9] = [1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                            2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                            2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]
            xf[t, b, 9:] = rng.standard_normal(3)
    return xf


def random_tree(J, seed=0):
    rng = np.random.default_rng(seed)
    parent = np.array([-1] + [int(rng.integers(0, k)) for k in range(1, J)])
    # depth-first renumbering
    kids = [[] for _ in range(J)]
    for k in range(1, J):
        kids[parent[k]].append(k)
    order, stack = [], [0]
    while stack:
        k = stack.pop()
        order.append(k)
        stack += kids[k][::-1]
    pos = np.empty(J, np.int64)
    pos[order] = np.arange(J)
    return np.array([-1] + [pos[parent[order[k]]] for k in range(1, J)])


def check_kernels(rest, faces, joints, weights, B, T, seed=0):
    count, prior = ops.autorig_pair_stats(_cuda(rest), _cuda(faces), _cuda(joints), _cuda(weights), B)
    rc, rp = ref.pair_stats(rest, faces, joints, weights, B)
    assert _same(count.cpu().numpy(), rc) and _same(prior.cpu().numpy(), rp)
    assert _same(ops.autorig_bone_weights(_cuda(joints), _cuda(weights), B).cpu().numpy(),
                 ref.bone_weights(joints, weights, B))
    xf = random_transforms(T, B, seed)
    centres = np.random.default_rng(seed).standard_normal((B, 3))
    pj, cost = ops.autorig_joint_solve(_cuda(xf), _cuda(centres), count, prior, autorig.LAMBDA)
    rj, re = ref.joint_solve(xf, centres, rc, rp)
    assert _same(pj.cpu().numpy(), rj) and _same(cost.cpu().numpy(), re)
    check_lists(rest, joints, weights, B, seed)


def check_lists(rest, joints, weights, J, seed=0):
    V = len(rest)
    parent = random_tree(J, seed)
    a = autorig.rig_layout(parent, np.zeros((J, 3)), rest)
    t = rigmod.rig_tensors(a, 1, torch.device("cuda"))
    ops.autorig_slots(_cuda(joints), _cuda(weights), t.slot_bind, t.slot_weight)
    sb, sw = ref.slots(joints, weights)
    assert _same(t.slot_bind.cpu().numpy(), sb) and _same(t.slot_weight.cpu().numpy(), sw)
    cap = autorig.list_capacity(parent, V)
    lists = torch.full((cap,), -7, dtype=torch.int32, device="cuda")
    offsets = torch.empty(J + 1, dtype=torch.int32, device="cuda")
    ops.autorig_joint_lists(t, _cuda(a.subtree_end.astype(np.int32)), lists, offsets)
    rl, ro = ref.joint_lists(np.arange(J), sb, sw, a.subtree_end)
    off = offsets.cpu().numpy()
    assert _same(off.astype(np.int64), ro) and _same(lists.cpu().numpy()[:off[J]], rl)
    # the host loop of rig.rig_arrays gives the same lists
    a.slot_bind, a.slot_weight = sb, sw
    host = rigmod.rig_arrays(type("R", (), dict(order=np.arange(J), parent=parent, above=np.tile(np.eye(4), (J, 1, 1)),
                                                 bind_joint=np.arange(J), slot_bind=sb, slot_weight=sw, scale=a.scale,
                                                 binds=np.tile(np.eye(4), (J, 1, 1)), rotation=np.tile([0, 0, 0, 1.0], (J, 1)),
                                                 translation=a.translations, points=rest, rest=rest))())
    assert np.array_equal(host.lists, rl) and np.array_equal(host.offsets, ro)


@pytest.mark.parametrize("V,B,T", [(5, 1, 2), (300, 2, 3), (700, 5, 4), (3000, 33, 3)])
def test_kernels_match_restatement(amb_lib, V, B, T):
    rest, faces = grid_mesh(V)
    joints, weights = random_skin(rest, B)
    check_kernels(rest, faces, joints, weights, B, T)


@pytest.mark.parametrize("V,B", [(20000, 32), (200000, 256)])
def test_kernels_at_production_sizes(amb_lib, V, B):
    rest, faces = grid_mesh(V)
    joints, weights = random_skin(rest, B, seed=1)
    check_kernels(rest, faces, joints, weights, B, 31, seed=1)


def test_whole_fit_matches_restatement_and_is_deterministic(amb_lib):
    rest, faces, W = syn.mesh(step=0.1, around=6)
    v, _ = syn.animate(rest, W, T=3)
    fits = [autorig.fit_auto_rig(v, faces, 7, rounds=2, sweeps=3) for _ in range(2)]
    r = ref.fit(v, faces, 7, rounds=2, sweeps=3)
    for f in fits:
        assert np.array_equal(f.parent, r["parent"]) and np.array_equal(f.bones, r["bones"])
        assert _same(f.positions, r["positions"])
        assert _same(f.rotation_matrices.reshape(3, 7, 9), r["rotations"])
        assert _same(f.root_translations, r["translations"][:, 0])
        assert _same(f.joints, r["joints"]) and _same(f.weights, r["weights"])
        assert _same(f.history, r["history"])


@pytest.mark.parametrize("V,J", [(20000, 32), (200000, 256)])
def test_production_rounds_replayed(amb_lib, V, J):
    """fit_auto_rig's own steps at production size, 31 frames: the pair tables, joint solve, tree, joint positions and warm
    start from the real SSDR fit; then, from the GPU's state after one whole round and the sweeps of the next, the weight
    half replayed: the skinning transforms K = G B, the new weights (restated per vertex, on every 25th vertex: each
    vertex's update reads only its own row), the rig's slots and lists over every vertex, and the error after it."""
    import rig_ref
    import skinning_ref

    step, around = {20000: (0.01, 50), 200000: (0.003, 152)}[V]
    rest, faces, W = syn.mesh(step=step, around=around)
    v, _ = syn.animate(rest, W, T=31, seed=2)
    T = v.shape[0]
    faces = faces.astype(np.int32)
    with torch.cuda.device(0):
        st = autorig.start_auto_rig(v, faces, J, torch.device("cuda", 0))
    sk = st.sk
    xf = np.concatenate([sk.rotations.reshape(T, J, 9), sk.translations], -1)
    rc, rp = ref.pair_stats(rest, faces, sk.joints, sk.weights, J)
    assert _same(st.pair_count, rc)
    assert _same(st.bone_weight, ref.bone_weights(sk.joints, sk.weights, J))
    rj, re = ref.joint_solve(xf, sk.centres, rc, rp)
    assert _same(st.pair_joint, rj) and _same(st.pair_cost, re)
    bones, parent, pair = ref.topology(rc, re, st.bone_weight)
    assert np.array_equal(st.bones, bones) and np.array_equal(st.parent, parent)
    c = np.stack([rj[p] if p >= 0 else sk.centres[b] for b, p in zip(bones, pair)])
    assert _same(st.positions, c)
    r0, t0 = ref.warm_start(xf, bones, parent, c)
    assert _same(st.rot.cpu().numpy(), r0) and _same(st.trans.cpu().numpy(), t0)

    autorig.sweep_half(st, autorig.DEFAULT_SWEEPS)
    autorig.weight_half(st)
    autorig.sweep_half(st, autorig.DEFAULT_SWEEPS)
    rot, trans = st.rot.cpu().numpy(), st.trans.cpu().numpy()
    joints, weights = st.joints.cpu().numpy(), st.weights.cpu().numpy()
    autorig.weight_half(st)
    a = st.a
    _, skin = rig_ref.forward(a, rot, trans)
    assert _same(st.t.skin.cpu().numpy(), skin)
    rows = np.arange(0, len(rest), 25)
    _, _, cand = skinning_ref.rigid_error(rest[rows], v[:, rows], skin)
    want_j, want_w = skinning_ref.weight_update(rest[rows], v[:, rows], skin, cand, joints[rows], weights[rows])
    new_j, new_w = st.joints.cpu().numpy(), st.weights.cpu().numpy()
    assert _same(new_j[rows], want_j) and _same(new_w[rows], want_w)
    sb, sw = ref.slots(new_j, new_w)
    assert _same(st.t.slot_bind.cpu().numpy(), sb) and _same(st.t.slot_weight.cpu().numpy(), sw)
    rl, ro = ref.joint_lists(np.arange(J), sb, sw, a.subtree_end)
    off = st.offsets.cpu().numpy()
    assert _same(off.astype(np.int64), ro) and _same(st.lists.cpu().numpy()[:off[J]], rl)
    a.slot_bind, a.slot_weight, a.lists, a.offsets = sb, sw, rl, ro
    frame_errors, _ = ops.rig_error(st.t, st.rot, st.trans, st.verts)
    assert _same(frame_errors.cpu().numpy(), rig_ref.error(a, rot, trans, v)[0])


def test_synthetic_skeleton_is_recovered(amb_lib):
    rest, faces, W = syn.mesh()
    v, _ = syn.animate(rest, W, T=6)
    fit = autorig.fit_auto_rig(v, faces, 7)
    diag = np.linalg.norm(rest.max(0) - rest.min(0))
    seg = syn.segment_of_bones(fit, W)
    assert syn.tree_edges(fit, seg) == syn.true_edges()
    assert syn.joint_errors(fit, seg).max() <= 1e-3 * diag
    assert fit.rms_error <= syn.RMS_BOUND
    h = fit.history
    assert all(h[i + 1] <= h[i] * (1 + 1e-12) for i in range(len(h) - 1))


@pytest.mark.parametrize("with_mesh", [False, True])
def test_end_to_end_on_the_tiny_tree(tmp_path, amb_lib, with_mesh):
    """auto_rig_joints adds only auto_rigged_mesh.glb, every other file and video frame equals a run without it, and the
    file decodes to the fit's M v^."""
    import standalone_tree as st
    from actionmesh_b200.gltf import ANIMATED_GLB_MAP, write_glb
    from actionmesh_b200.inference import run_actionmesh
    from actionmesh_b200.pipeline import ActionMeshB200Pipeline, ActionMeshB200PipelineWithMeshInput, Mesh
    from test_inference_gpu import UPDATES, _frames_dir, _video_frames

    frames = _frames_dir(tmp_path, 16)
    root = st.centred_tree(str(tmp_path / "pretrained_weights"))
    kw = {}
    if with_mesh:
        rest, faces, _ = syn.mesh(step=0.1, around=8)
        path = tmp_path / "plain.glb"
        write_glb(path, Mesh(vertices=rest * 0.3, faces=faces))
        kw["mesh_input"] = str(path)
        updates = {**UPDATES, "model.temporal_3D_denoiser.num_tokens_nominal": 2048}
        pipe = ActionMeshB200PipelineWithMeshInput.from_pretrained(root, config_updates=updates).to("cuda")
    else:
        pipe = ActionMeshB200Pipeline.from_pretrained(root, config_updates=UPDATES).to("cuda")
    outs = [tmp_path / "plain", tmp_path / "auto"]
    run_actionmesh(pipe, str(frames), str(outs[0]), seed=44, **kw)
    meshes = run_actionmesh(pipe, str(frames), str(outs[1]), seed=44, auto_rig_joints=4, **kw)
    names = sorted(p.name for p in outs[0].iterdir())
    assert sorted(p.name for p in outs[1].iterdir()) == sorted(names + ["auto_rigged_mesh.glb"])
    for name in names:
        if name.endswith(".mp4"):
            assert np.array_equal(_video_frames(outs[0] / name), _video_frames(outs[1] / name))
        else:
            assert (outs[0] / name).read_bytes() == (outs[1] / name).read_bytes(), name
    vertices = np.stack([np.asarray(m.vertices) for m in meshes])
    faces = np.asarray(meshes[0].faces)
    fit = autorig.fit_auto_rig(vertices, faces, 4)
    want = autorig.posed_vertices(fit) @ ANIMATED_GLB_MAP.T
    out = outs[1] / "auto_rigged_mesh.glb"
    glb_check.check_glb(out)
    for k in range(len(vertices)):
        assert np.abs(evaluate(out, key=k) - want[k]).max() <= 2.0 ** -18 * max(1.0, np.abs(want).max()), k
