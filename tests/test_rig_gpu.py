"""The rig fit on the GPU (-m gpu), bit for bit against tests/rig_ref.py.

- Kernel by kernel on 1-, 3- and 65-joint rigs: forward kinematics, the rotation and translation updates of every joint
  (empty subtrees, vertices on a pivot), the error sums.
- Whole small fits, and two runs of one fit.
- Production sizes: 20 000 and 200 000 vertices x 31 frames x 65 joints, with the first, a middle and the last sweep
  replayed through the restatement from the GPU's own state.
- The command line's path on the tiny checkpoint tree with a rigged mesh input and keep_rig."""
import numpy as np
import pytest
import torch

import glb_check
import rig_ref as ref
from actionmesh_b200 import rig as rigmod
from test_rig_cpu import animation, evaluate, rigged_file, synthetic_rig

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _mat4(monkeypatch):
    """glb_check reads the vector accessor types; a skin's inverse bind matrices are MAT4 (16 components)."""
    monkeypatch.setitem(glb_check.NCOMP, "MAT4", 16)


def _same(a, b) -> bool:
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype == np.float64:
        return a.shape == b.shape and np.array_equal(a.view(np.uint64), np.asarray(b, np.float64).view(np.uint64))
    return a.shape == b.shape and np.array_equal(a, b)


def _cuda(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def random_rig(J, V, T, seed=0, empty=(), pivot=True):
    """RigArrays of a random J-joint tree (parents before children, depth-first), its vertices skinned to up to 8 joints
    near each other, rigid-child binds, a few static vertices and vertices exactly on a joint's pivot; joints in `empty`
    influence nothing.  -> (arrays, rotations (T, J, 9), translations (T, J, 3), vertices (T, V, 3))."""
    rng = np.random.default_rng(seed)
    parent = [-1]
    for j in range(1, J):
        parent.append(int(rng.integers(max(0, j - 4), j)) if j % 9 else -1)
    # depth-first renumbering
    kids = [[] for _ in range(J)]
    for j in range(1, J):
        if parent[j] >= 0:
            kids[parent[j]].append(j)
    order, stack = [], [j for j in range(J - 1, -1, -1) if parent[j] < 0]
    while stack:
        j = stack.pop()
        order.append(j)
        stack.extend(reversed(kids[j]))
    q = np.stack([rigmod._rotation_matrix(x) for x in rng.standard_normal((J, 4))])
    xf = lambda lin, t: np.concatenate([lin.reshape(-1, 9), t.reshape(-1, 3)], 1)
    above = xf(np.stack([0.5 * np.linalg.qr(rng.standard_normal((3, 3)))[0] for _ in range(J)]), rng.standard_normal((J, 3)))
    above[:, :9] *= np.where(np.linalg.det(above[:, :9].reshape(J, 3, 3)) < 0, -1, 1)[:, None]
    NB = J + 3
    binds = xf(np.eye(3)[None] + 0.1 * rng.standard_normal((NB, 3, 3)), rng.standard_normal((NB, 3)))
    bind_joint = np.concatenate([np.arange(J), rng.integers(0, J, 3)])
    live = np.array([b for b in range(NB) if bind_joint[b] not in empty])
    sb, sw = np.zeros((V, 8), np.int32), np.zeros((V, 8))
    for i in range(V):
        n = 1 + i % 8
        if i % 50 == 7:
            continue                                      # static
        sb[i, :n] = rng.choice(live, n, replace=False) if n <= len(live) else rng.choice(live, n)
        w = rng.uniform(0.1, 1, n)
        sw[i, :n] = w / w.sum()
    points = rng.standard_normal((V, 3))
    if pivot:
        # vertices on joint 0's pivot: their bind maps them to the joint's origin
        points[1:4] = -binds[0, 9:]
        binds[0, :9] = np.eye(3).ravel()
        sb[1:4, 0], sw[1:4] = 0, 0
        sw[1:4, 0] = 1.0
    rig = type("Rig", (), {})()
    rig.order = np.array(order)
    rig.parent = np.array(parent)
    rig.scale = np.where(rng.uniform(size=(J, 1)) < 0.5, 1.0, rng.uniform(0.5, 2, (J, 1))) * np.ones((J, 3))
    rig.above = np.tile(np.eye(4), (J, 1, 1))
    rig.above[:, :3, :3] = above[:, :9].reshape(J, 3, 3)
    rig.above[:, :3, 3] = above[:, 9:]
    rig.binds = np.tile(np.eye(4), (NB, 1, 1))
    rig.binds[:, :3, :3] = binds[:, :9].reshape(NB, 3, 3)
    rig.binds[:, :3, 3] = binds[:, 9:]
    rig.bind_joint = bind_joint
    rig.rotation = rng.standard_normal((J, 4))
    rig.rotation /= np.linalg.norm(rig.rotation, axis=1, keepdims=True)
    rig.translation = rng.standard_normal((J, 3))
    rig.points, rig.rest = points, rng.standard_normal((V, 3))
    rig.slot_bind, rig.slot_weight = sb, sw
    a = rigmod.rig_arrays(rig)
    rots = np.ascontiguousarray(np.broadcast_to(a.rotations, (T, J, 9))).copy()
    for t in range(T):
        for j in range(J):
            rots[t, j] = (rots[t, j].reshape(3, 3) @ rigmod._rotation_matrix(
                np.concatenate([0.3 * rng.standard_normal(3), [1.0]]))).ravel()
    trs = np.ascontiguousarray(np.broadcast_to(a.translations, (T, J, 3))).copy()
    trs[:, a.parent < 0] += 0.2 * rng.standard_normal((T, int((a.parent < 0).sum()), 3))
    verts = ref.posed(a, rots, trs) + 0.01 * rng.standard_normal((T, V, 3))
    return a, rots, trs, verts


def _tensors(a, T):
    return rigmod.rig_tensors(a, T, torch.device("cuda", torch.cuda.current_device()))


@pytest.mark.parametrize("J,V,T", [(1, 300, 3), (3, 700, 4), (65, 3000, 3)])
def test_kernels_match_restatement(amb_lib, J, V, T):
    from actionmesh_b200 import ops

    a, rots, trs, verts = random_rig(J, V, T, seed=J, empty=(J - 1,) if J > 1 else ())
    t = _tensors(a, T)
    r, tr, vv = _cuda(rots), _cuda(trs), _cuda(verts)
    ops.rig_forward(t, r, tr)
    world, skin = ref.forward(a, rots, trs)
    assert _same(t.world.cpu().numpy(), world) and _same(t.skin.cpu().numpy(), skin)
    fe, mx = (x.cpu().numpy() for x in ops.rig_error(t, r, tr, vv))
    wfe, wmx = ref.error(a, rots, trs, verts)
    assert _same(fe, wfe) and _same(mx, np.array([wmx]))
    lists = _cuda(a.lists)
    for k in range(J):
        lst = a.lists[a.offsets[k]:a.offsets[k + 1]]
        end = int(a.subtree_end[k])
        ops.rig_rotation_update(t, r, tr, vv, lists[int(a.offsets[k]):int(a.offsets[k + 1])], k, end)
        rots = ref.rotation_update(a, rots, trs, verts, lst, k, end)
        assert _same(r.cpu().numpy(), rots), k
        if a.parent[k] < 0:
            ops.rig_translation_update(t, r, tr, vv, lists[int(a.offsets[k]):int(a.offsets[k + 1])], k, end)
            trs = ref.translation_update(a, rots, trs, verts, lst, k, end)
            assert _same(tr.cpu().numpy(), trs), k
    if J > 1:
        leaf = int(np.flatnonzero(a.order == J - 1)[0])
        assert a.offsets[leaf] == a.offsets[leaf + 1]           # the empty leaf had no list and kept its rotation


def _file_rig(tmp_path, V=300, T=3):
    from actionmesh_b200.gltf import load_rig

    path = tmp_path / "rigged.glb"
    rigged_file(path, V=V)
    rig = load_rig(path)
    a, rots, trs = animation(rig, T)
    return path, rig, a, ref.posed(a, rots, trs)


def test_whole_fit_matches_restatement_and_is_deterministic(amb_lib, tmp_path):
    path, rig, a, verts = _file_rig(tmp_path)
    fit = rigmod.fit_rig_animation(rig, verts, sweeps=3)
    rot, trans, history = ref.fit(a, verts, 3)
    T, J = rot.shape[:2]
    assert _same(fit.rotation_matrices[:, a.order].reshape(T, J, 9), rot)
    assert _same(fit.translations[:, a.order], trans)
    assert _same(np.array(fit.history), np.array(history))
    again = rigmod.fit_rig_animation(rig, verts, sweeps=3)
    assert _same(again.rotation_matrices, fit.rotation_matrices) and _same(again.translations, fit.translations)
    assert again.history == fit.history and again.rms_error == fit.rms_error and again.max_error == fit.max_error


def test_default_sweeps_recover_an_exact_animation(amb_lib):
    rig, a, verts = synthetic_rig()
    fit = rigmod.fit_rig_animation(rig, verts)
    assert fit.rms_error <= 1e-6, fit.history
    assert all(b <= x * (1 + 1e-12) for x, b in zip(fit.history, fit.history[1:]))


def test_written_file_shows_the_fit(amb_lib, tmp_path):
    from actionmesh_b200.gltf import write_rig_animation

    path, rig, a, verts = _file_rig(tmp_path, V=240, T=3)
    fit = rigmod.fit_rig_animation(rig, verts, sweeps=10)
    out = tmp_path / "rigged_mesh.glb"
    write_rig_animation(path, out, rig, fit)
    want = ref.posed(a, fit.rotation_matrices[:, a.order].reshape(3, -1, 9), fit.translations[:, a.order])
    for k in range(3):
        assert np.abs(evaluate(out, key=k) - want[k]).max() <= 2.0 ** -18 * max(1.0, np.abs(want).max()), k


# ---- production sizes --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V", [20000, 200000])
def test_production_sweeps_replayed(amb_lib, V):
    """65 joints x 31 frames: sweeps 0, 2 and 4 of 5 replayed from the GPU's state.  Every fourth joint's update and every
    root's is checked at 20 000 vertices; joints 0, 32 and 64 and the roots at 200 000; the error sums on every vertex."""
    from actionmesh_b200 import ops

    T, J = 31, 65
    a, _, _, verts = random_rig(J, V, T, seed=7, empty=(40,))
    check = set(range(0, J, 4) if V <= 20000 else (0, 32, 64)) | set(np.flatnonzero(a.parent < 0).tolist())
    lists = _cuda(a.lists)
    vv = _cuda(verts)
    for s_idx in (0, 2, 4):
        t = _tensors(a, T)
        # the GPU's state after s_idx sweeps, through the driver's own loop
        r = _cuda(np.broadcast_to(a.rotations, (T, J, 9)))
        tr = _cuda(np.broadcast_to(a.translations, (T, J, 3)))
        for s in range(s_idx + 1):
            for k in range(J):
                end = int(a.subtree_end[k])
                lst = lists[int(a.offsets[k]):int(a.offsets[k + 1])]
                before = (r.cpu().numpy(), tr.cpu().numpy()) if s == s_idx and k in check else None
                ops.rig_rotation_update(t, r, tr, vv, lst, k, end)
                if before is not None:
                    want = ref.rotation_update(a, before[0], before[1], verts, a.lists[a.offsets[k]:a.offsets[k + 1]], k, end)
                    assert _same(r.cpu().numpy()[:, k], want[:, k]), (s, k)
                if a.parent[k] < 0:
                    before = (r.cpu().numpy(), tr.cpu().numpy()) if s == s_idx and k in check else None
                    ops.rig_translation_update(t, r, tr, vv, lst, k, end)
                    if before is not None:
                        want = ref.translation_update(a, before[0], before[1], verts,
                                                      a.lists[a.offsets[k]:a.offsets[k + 1]], k, end)
                        assert _same(tr.cpu().numpy()[:, k], want[:, k]), (s, k)
        fe, mx = (x.cpu().numpy() for x in ops.rig_error(t, r, tr, vv))
        wfe, wmx = ref.error(a, r.cpu().numpy(), tr.cpu().numpy(), verts)
        assert _same(fe, wfe) and _same(mx, np.array([wmx])), s_idx


# ---- the command line's path -------------------------------------------------------------------------------------------------
def test_rigged_mesh_input_end_to_end(tmp_path, amb_lib):
    """A hand-built rigged GLB as the mesh input on the tiny checkpoint tree: rigged_mesh.glb decodes to the fit's v^, and
    every other file is the one a run without the rig writes."""
    import standalone_tree as st
    from actionmesh_b200.gltf import load_rig
    from actionmesh_b200.inference import run_actionmesh
    from actionmesh_b200.pipeline import ActionMeshB200PipelineWithMeshInput
    from test_inference_gpu import UPDATES, _frames_dir, _video_frames

    mesh = tmp_path / "rigged.glb"
    rigged_file(mesh, V=600)
    rig = load_rig(mesh)
    frames = _frames_dir(tmp_path, 16)
    root = st.centred_tree(str(tmp_path / "pretrained_weights"))
    updates = {**UPDATES, "model.temporal_3D_denoiser.num_tokens_nominal": 2048}
    pipe = ActionMeshB200PipelineWithMeshInput.from_pretrained(root, config_updates=updates).to("cuda")
    outs = [tmp_path / "plain", tmp_path / "rig"]
    run_actionmesh(pipe, str(frames), str(outs[0]), seed=44, mesh_input=str(mesh))
    meshes = run_actionmesh(pipe, str(frames), str(outs[1]), seed=44, mesh_input=str(mesh), rig=rig)
    names = sorted(p.name for p in outs[0].iterdir())
    assert sorted(p.name for p in outs[1].iterdir()) == sorted(names + ["rigged_mesh.glb"])
    for name in names:
        if name.endswith(".mp4"):
            assert np.array_equal(_video_frames(outs[0] / name), _video_frames(outs[1] / name))
        else:
            assert (outs[0] / name).read_bytes() == (outs[1] / name).read_bytes(), name
    vertices = np.stack([np.asarray(m.vertices) for m in meshes])
    fit = rigmod.fit_rig_animation(rig, vertices)
    a = rigmod.rig_arrays(rig)
    T = len(vertices)
    want = ref.posed(a, fit.rotation_matrices[:, a.order].reshape(T, -1, 9), fit.translations[:, a.order])
    out = outs[1] / "rigged_mesh.glb"
    glb_check.check_glb(out)
    for k in range(T):
        assert np.abs(evaluate(out, key=k) - want[k]).max() <= 2.0 ** -18 * max(1.0, np.abs(want).max()), k

