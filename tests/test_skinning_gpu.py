"""The skinning decomposition on the GPU (-m gpu), bit for bit against tests/skinning_ref.py.

- Kernel by kernel on small cases: seeds (with repeated points), rigid errors and candidates (B below and above 8), the bone
  update of every bone (empty bones, 1- and 2-vertex bones), the weight update (bones with identical transforms: exact ties and
  singular subsets), the error sums.
- Whole fits at small sizes, and two runs of one fit.
- Production sizes: 20 000 and 200 000 vertices x 31 frames x 32 bones, with the first, a middle and the last iteration
  replayed through the restatement from the GPU's own state.
- The command line's path on the tiny checkpoint tree with skinning_bones=16."""
import numpy as np
import pytest
import torch

import glb_check
import skinning_ref as ref
from test_skinning_cpu import bent_cylinder, check_skinned, rigid_parts

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


def _cuda(*arrays):
    return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]


def _random_state(V=700, T=5, B=12, seed=0):
    """Random rest / vertices / transforms (rotations near the identity) and <= 4-slot weights with empty bones, one
    1-vertex bone and one 2-vertex bone."""
    rng = np.random.default_rng(seed)
    rest = rng.standard_normal((V, 3))
    verts = rest[None] + 0.2 * rng.standard_normal((T, V, 3))
    verts[0] = rest
    xf = np.zeros((T, B, 12))
    for t in range(T):
        for j in range(B):
            q, r = np.linalg.qr(np.eye(3) + 0.3 * rng.standard_normal((3, 3)))
            q = q * np.sign(np.diag(r))
            xf[t, j, :9] = (q if np.linalg.det(q) > 0 else -q).ravel()
            xf[t, j, 9:] = 0.1 * rng.standard_normal(3)
    joints = np.zeros((V, 4), np.int32)
    weights = np.zeros((V, 4))
    live = B - 4                                   # bones B-4 .. B-1: B-4 and B-3 empty, B-2 one vertex, B-1 two
    for i in range(V):
        n = 1 + i % 4
        joints[i, :n] = rng.choice(live, n, replace=False)
        w = rng.uniform(0.1, 1.0, n)
        weights[i, :n] = w / w.sum()
    joints[5], weights[5] = [B - 2, 0, 0, 0], [1.0, 0, 0, 0]
    joints[6], weights[6] = [B - 1, 1, 0, 0], [0.25, 0.75, 0, 0]
    joints[7], weights[7] = [2, B - 1, 0, 0], [0.5, 0.5, 0, 0]
    joints[8], weights[8] = [1, 3, 4, 0], [0.5, 0.0, 0.5, 0.0]      # a zero weight between used slots
    return rest, verts, xf, joints, weights


def test_seeds_match_restatement(amb_lib):
    from actionmesh_b200 import ops

    rng = np.random.default_rng(1)
    rest = rng.standard_normal((5000, 3))
    rest[100:200] = rest[0]                      # repeated points: ties go to the lowest index
    rest[300] = rest[3000]
    for B in (1, 7, 64, 256):
        seeds, labels, centres = (t.cpu().numpy() for t in ops.skin_seeds(*_cuda(rest), B))
        ws, wl, wc = ref.seeds(rest, B)
        assert _same(seeds, ws) and _same(labels, wl) and _same(centres, wc), B


@pytest.mark.parametrize("B", [3, 8, 12])
def test_rigid_error_matches_restatement(amb_lib, B):
    from actionmesh_b200 import ops

    rest, verts, xf, _, _ = _random_state()
    xf = xf[:, :B].copy()
    xf[:, B - 1] = xf[:, 0]                      # equal errors: the lower bone index first
    got = [t.cpu().numpy() for t in ops.skin_rigid_error(*_cuda(rest, verts, xf))]
    want = ref.rigid_error(rest, verts, xf)
    for g, w in zip(got, want):
        assert _same(g, w)


def test_bone_update_matches_restatement_for_every_bone(amb_lib):
    from actionmesh_b200 import ops

    rest, verts, xf, joints, weights = _random_state()
    B = xf.shape[1]
    centres = np.arange(3 * B, dtype=np.float64).reshape(B, 3)
    r, v, x, j, w, c = _cuda(rest, verts, xf, joints, weights, centres)
    for bone in range(B):
        ops.skin_bone_update(r, v, x, j, w, bone, c)
        xf, centres = ref.bone_update(rest, verts, xf, joints, weights, bone, centres)
        assert _same(x.cpu().numpy(), xf) and _same(c.cpu().numpy(), centres), bone
    # empty bones keep their transform and centre
    assert _same(centres[B - 4], np.arange(3 * (B - 4), 3 * (B - 3), dtype=np.float64))


def test_bone_update_of_a_rigid_cluster_is_exact(amb_lib):
    """One-hot weights on a rigidly moving cluster: Kabsch recovers the motion to rounding."""
    from actionmesh_b200 import ops

    v = rigid_parts(n_parts=1, n_per_part=50, frames=4)
    V = v.shape[1]
    xf = np.zeros((4, 1, 12))
    xf[:, :, [0, 4, 8]] = 1.0
    joints, weights = np.zeros((V, 4), np.int32), np.zeros((V, 4))
    weights[:, 0] = 1.0
    r, vv, x, j, w = _cuda(v[0], v, xf, joints, weights)
    c = torch.zeros(1, 3, dtype=torch.float64, device="cuda")
    ops.skin_bone_update(r, vv, x, j, w, 0, c)
    fe, _ = ops.skin_error(r, vv, x, j, w)
    assert float(fe[-1]) <= 1e-24 * V * 4


def test_weight_update_matches_restatement(amb_lib):
    from actionmesh_b200 import ops

    rest, verts, xf, joints, weights = _random_state(V=1500, B=12)
    xf[:, 3] = xf[:, 2]                          # identical bones: exact ties and singular subsets
    xf[:, 5] = xf[:, 2]
    _, _, cand = ops.skin_rigid_error(*_cuda(rest, verts, xf))
    cand = cand.cpu().numpy()
    r, v, x, cd, j, w = _cuda(rest, verts, xf, cand, joints, weights)
    ops.skin_weight_update(r, v, x, cd, j, w)
    wj, ww = ref.weight_update(rest, verts, xf, cand, joints, weights)
    assert _same(j.cpu().numpy(), wj) and _same(w.cpu().numpy(), ww)
    assert (ww >= 0).all() and (np.count_nonzero(ww, 1) >= 1).all()


def test_error_matches_restatement(amb_lib):
    from actionmesh_b200 import ops

    for V in (12, 255, 257, 3000):
        rest, verts, xf, joints, weights = _random_state(V=V, seed=V)
        fe, mx = (t.cpu().numpy() for t in ops.skin_error(*_cuda(rest, verts, xf, joints, weights)))
        wfe, wmx = ref.error(rest, verts, xf, joints, weights)
        assert _same(fe, wfe) and _same(mx, np.array([wmx])), V


@pytest.mark.parametrize("case", ["cylinder_8", "cylinder_3", "rigid_4"])
def test_whole_fit_matches_restatement(amb_lib, case):
    from actionmesh_b200.skinning import fit_skinning

    v, B = {"cylinder_8": (bent_cylinder(), 8), "cylinder_3": (bent_cylinder(frames=3), 3),
            "rigid_4": (rigid_parts(), 4)}[case]
    fit = fit_skinning(v, B, iterations=4)
    want = ref.fit(v, B, 4)
    T = v.shape[0]
    assert _same(fit.rotations.reshape(T, B, 9), want["transforms"][:, :, :9])
    assert _same(fit.translations, want["transforms"][:, :, 9:])
    assert _same(fit.joints, want["joints"]) and _same(fit.weights, want["weights"])
    assert _same(fit.centres, want["centres"])
    assert _same(np.array(fit.history), np.array(want["history"]))


def test_fit_is_deterministic(amb_lib):
    from actionmesh_b200.skinning import fit_skinning

    v = _animated_blob(20000, seed=5)
    a, b = fit_skinning(v, 32, iterations=3), fit_skinning(v, 32, iterations=3)
    for name in ("rotations", "translations", "joints", "weights", "centres"):
        assert _same(getattr(a, name), getattr(b, name)), name
    assert a.history == b.history and a.rms_error == b.rms_error and a.max_error == b.max_error


# ---- production sizes --------------------------------------------------------------------------------------------------------
def _animated_blob(V, T=31, seed=0) -> np.ndarray:
    """(T, V, 3): points on a bumpy closed surface, bent, twisted and translated smoothly over the frames."""
    rng = np.random.default_rng(seed)
    d = rng.standard_normal((V, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    rest = d * (1 + 0.2 * np.sin(3 * d[:, :1]) * np.cos(2 * d[:, 1:2])) * np.array([0.6, 0.6, 1.5])
    out = []
    for t in range(T):
        s = t / max(T - 1, 1)
        a = 0.8 * s * rest[:, 2:3]                # twist about z, growing with height
        x = rest[:, :1] * np.cos(a) - rest[:, 1:2] * np.sin(a)
        y = rest[:, :1] * np.sin(a) + rest[:, 1:2] * np.cos(a)
        z = rest[:, 2:3]
        x = x + 0.3 * s * z ** 2                  # bend
        out.append(np.concatenate([x, y, z], 1) + np.array([0.1 * s, 0.0, 0.05 * np.sin(3 * s)]))
    return np.stack(out)


def _state(fit):
    T, B = fit.rotations.shape[:2]
    xf = np.concatenate([fit.rotations.reshape(T, B, 9), fit.translations], 2)
    return xf, fit.joints.copy(), fit.weights.copy(), fit.centres.copy()


@pytest.mark.parametrize("V", [20000, 200000])
def test_production_iterations_replayed(amb_lib, V):
    """A 32-bone fit of 31 frames: iterations 0, 4 and 7 of 8 replayed from the GPU's state.  Every bone update is checked
    at 20 000 vertices, bones 0, 15 and 31 at 200 000; the rigid errors and the weight update on every vertex at 20 000 and
    on 4 000 sampled vertices at 200 000; the error sums on every vertex."""
    from actionmesh_b200 import ops
    from actionmesh_b200.skinning import fit_skinning

    v = _animated_blob(V)
    rest = v[0]
    B, T = 32, v.shape[0]
    bones = range(B) if V <= 20000 else (0, 15, 31)
    sample = np.arange(V) if V <= 20000 else np.sort(np.random.default_rng(0).choice(V, 4000, replace=False))
    last = None
    for it in (0, 4, 7):
        xf, joints, weights, centres = _state(fit_skinning(v, B, iterations=it))
        r, vv, x, j, w, c = _cuda(rest, v, xf, joints, weights, centres)
        for bone in range(B):
            before = (x.cpu().numpy(), c.cpu().numpy()) if bone in bones else None
            ops.skin_bone_update(r, vv, x, j, w, bone, c)
            if before is not None:
                wx, wc = ref.bone_update(rest, v, before[0], joints, weights, bone, before[1])
                assert _same(x.cpu().numpy()[:, bone], wx[:, bone]) and _same(c.cpu().numpy()[bone], wc[bone]), (it, bone)
        xf_new = x.cpu().numpy()
        argmin, min_err, cand = (t.cpu().numpy() for t in ops.skin_rigid_error(r, vv, x))
        vs = np.ascontiguousarray(v[:, sample])
        wa, wm, wcand = ref.rigid_error(rest[sample], vs, xf_new)
        assert _same(argmin[sample], wa) and _same(min_err[sample], wm) and _same(cand[sample], wcand), it
        ops.skin_weight_update(r, vv, x, _cuda(cand)[0], j, w)
        wj, ww = ref.weight_update(rest[sample], vs, xf_new, cand[sample], joints[sample], weights[sample])
        gj, gw = j.cpu().numpy(), w.cpu().numpy()
        assert _same(gj[sample], wj) and _same(gw[sample], ww), it
        fe, mx = (t.cpu().numpy() for t in ops.skin_error(r, vv, x, j, w))
        wfe, wmx = ref.error(rest, v, xf_new, gj, gw)
        assert _same(fe, wfe) and _same(mx, np.array([wmx])), it
        # the replayed iteration is the driver's next iteration
        nxf, nj, nw, nc = _state(fit_skinning(v, B, iterations=it + 1))
        assert _same(xf_new, nxf) and _same(gj, nj) and _same(gw, nw) and _same(c.cpu().numpy(), nc), it
        last = fe[T]
    fit = fit_skinning(v, B, iterations=8)
    assert fit.history[-1] == last
    assert all(b <= a for a, b in zip(fit.history, fit.history[1:])), fit.history
    assert fit.rms_error < 0.01, fit.rms_error


# ---- the command line's path -------------------------------------------------------------------------------------------------
def test_run_actionmesh_writes_the_skinned_glb(root, tmp_path):
    """skinning_bones=16 on the tiny checkpoint tree: skinned_mesh.glb shows the 16-bone fit of the animated GLB's vertices,
    and every other file is the one a run without it writes."""
    from actionmesh_b200.inference import run_actionmesh
    from actionmesh_b200.pipeline import ActionMeshB200Pipeline
    from actionmesh_b200.skinning import fit_skinning
    from test_inference_gpu import UPDATES, _frames_dir, _video_frames

    frames = _frames_dir(tmp_path, 16)
    pipe = ActionMeshB200Pipeline.from_pretrained(root, config_updates=UPDATES).to("cuda")
    outs = [tmp_path / "plain", tmp_path / "skinned"]
    run_actionmesh(pipe, str(frames), str(outs[0]), seed=44)
    meshes = run_actionmesh(pipe, str(frames), str(outs[1]), seed=44, skinning_bones=16)
    names = sorted(p.name for p in outs[0].iterdir())
    assert sorted(p.name for p in outs[1].iterdir()) == sorted(names + ["skinned_mesh.glb"])
    for name in names:
        if name.endswith(".mp4"):
            assert np.array_equal(_video_frames(outs[0] / name), _video_frames(outs[1] / name))
        else:
            assert (outs[0] / name).read_bytes() == (outs[1] / name).read_bytes(), name
    vertices = np.stack([np.asarray(m.vertices) for m in meshes])
    fit = fit_skinning(vertices, 16)
    check_skinned(outs[1] / "skinned_mesh.glb", fit, meshes[0].faces)


from test_inference_gpu import root  # noqa: E402,F401  (the tiny checkpoint tree)
