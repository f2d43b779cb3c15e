"""The skinning decomposition's rules and its file on the CPU: the numpy restatement (tests/skinning_ref.py) recovers
piecewise-rigid and smoothly skinned animations and never increases its error; `gltf.write_skinned_glb` writes a valid GLB
whose skin, read back by an independent evaluator, shows the fit's reconstruction at every keyframe; `fit_skinning` and the
writer refuse bad arguments; the command line's `--skinning_bones` writes skinned_mesh.glb and nothing else changes."""
import numpy as np
import pytest

import glb_check
import skinning_ref as ref
from actionmesh_b200.gltf import GltfVisual, write_skinned_glb
from actionmesh_b200.skinning import SkinningFit, fit_skinning


def _rotation(rng) -> np.ndarray:
    q, r = np.linalg.qr(rng.standard_normal((3, 3)))
    q = q * np.sign(np.diag(r))
    return q if np.linalg.det(q) > 0 else -q


def rigid_parts(n_parts=4, n_per_part=30, frames=6, seed=0) -> np.ndarray:
    """(T, V, 3): n_parts unit blobs 10 apart (further than their diameters), each moved by its own random rigid transform
    in every frame after the first."""
    rng = np.random.default_rng(seed)
    parts = [np.array([10.0 * k, 0.0, 0.0]) + rng.uniform(-1, 1, (n_per_part, 3)) for k in range(n_parts)]
    out = [np.concatenate(parts)]
    for _ in range(1, frames):
        out.append(np.concatenate([p @ _rotation(rng).T + rng.standard_normal(3) for p in parts]))
    return np.stack(out)


def bent_cylinder(frames=8, n_ring=12, n_len=20) -> np.ndarray:
    """(T, V, 3): a cylinder of radius 1 and length 3 bent by 3 bones about x, with smooth (Gaussian, normalised) weights."""
    th = np.linspace(0, 2 * np.pi, n_ring, endpoint=False)
    z = np.linspace(0, 3, n_len)
    p = np.stack([np.tile(np.cos(th), n_len), np.tile(np.sin(th), n_len), np.repeat(z, n_ring)], -1)
    centres = np.array([0.5, 1.5, 2.5])
    w = np.exp(-(p[:, 2:3] - centres) ** 2 / 0.3)
    w /= w.sum(1, keepdims=True)
    out = []
    for t in range(frames):
        out.append(np.zeros_like(p))
        for j in range(3):
            a = 0.5 * np.sin(np.pi * t / frames) * j
            R = np.array([[1, 0, 0], [0, np.cos(a), -np.sin(a)], [0, np.sin(a), np.cos(a)]])
            pivot = np.array([0.0, 0.0, centres[j] - 0.5])
            out[-1] += w[:, j:j + 1] * ((p - pivot) @ R.T + pivot)
    return np.stack(out)


def diagonal(v) -> float:
    return float(np.linalg.norm(v[0].max(0) - v[0].min(0)))


def rms(v, total) -> float:
    return float(np.sqrt(total / (v.shape[0] * v.shape[1]))) / diagonal(v)


def as_fit(v, r) -> SkinningFit:
    """A SkinningFit holding the restatement's result `r` for the animation `v`."""
    T, B = r["transforms"].shape[:2]
    return SkinningFit(rest=v[0].copy(), joints=r["joints"], weights=r["weights"],
                       rotations=r["transforms"][:, :, :9].reshape(T, B, 3, 3), translations=r["transforms"][:, :, 9:],
                       centres=r["centres"], history=r["history"], rms_error=rms(v, r["history"][-1]), max_error=0.0)


def reconstruct(fit) -> np.ndarray:
    """(T, V, 3) float64 sum_k w_k (R p + t) of the fit."""
    u = np.einsum("tbij,vj->tvbi", fit.rotations, fit.rest) + fit.translations[:, None]
    T, V = u.shape[:2]
    return np.einsum("vk,tvki->tvi", fit.weights, u[:, np.arange(V)[:, None], fit.joints])


def _quat_matrix(q) -> np.ndarray:
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def skinned_frames(path) -> dict:
    """Read a skinned GLB with the test reader and evaluate its linear blend skinning at every keyframe (glTF 2.0: joint
    matrix = the joint node's global transform times its inverse bind matrix) -> positions (K, V, 3), times, the JSON."""
    gltf, binary = glb_check.check_glb(path)
    acc = lambda i: glb_check.accessor(gltf, binary, i).astype(np.float64)  # noqa: E731
    node = gltf["nodes"][0]
    prim = gltf["meshes"][node["mesh"]]["primitives"][0]
    skin = gltf["skins"][node["skin"]]
    pos, jn, wt = acc(prim["attributes"]["POSITION"]), acc(prim["attributes"]["JOINTS_0"]).astype(int), \
        acc(prim["attributes"]["WEIGHTS_0"])
    ibm = acc(skin["inverseBindMatrices"]).reshape(-1, 4, 4).transpose(0, 2, 1)
    root = gltf["nodes"][skin["skeleton"]]
    assert not any(k in root for k in ("matrix", "translation", "rotation", "scale"))
    assert root["children"] == skin["joints"]
    anim = gltf["animations"][0]
    keys, times = {}, None
    for ch in anim["channels"]:
        smp = anim["samplers"][ch["sampler"]]
        assert smp["interpolation"] == "LINEAR"
        times = acc(smp["input"])[:, 0]
        keys[ch["target"]["node"], ch["target"]["path"]] = acc(smp["output"])
    out = []
    for k in range(len(times)):
        mats = []
        for j, n in enumerate(skin["joints"]):
            g = np.eye(4)
            g[:3, :3] = _quat_matrix(keys[n, "rotation"][k])
            g[:3, 3] = keys[n, "translation"][k]
            mats.append(g @ ibm[j])
        mats = np.stack(mats)
        hom = np.concatenate([pos, np.ones((len(pos), 1))], 1)
        out.append(np.einsum("vk,vkij,vj->vi", wt, mats[jn], hom)[:, :3])
    return {"positions": np.stack(out), "times": times, "gltf": gltf, "binary": binary, "weights": wt, "joints": jn,
            "faces": acc(prim["indices"]).astype(np.int64).reshape(-1, 3), "keys": keys}


def check_skinned(path, fit, faces, fps=8) -> dict:
    """Assert that the skinned GLB at `path` shows blender_frame(the fit's reconstruction) at every keyframe k / fps."""
    got = skinned_frames(path)
    want = glb_check.blender_frame(reconstruct(fit))
    assert got["positions"].shape == want.shape
    tol = 2.0 ** -18 * max(1.0, np.abs(want).max())
    err = np.abs(got["positions"] - want).max()
    assert err <= tol, (err, tol)
    assert np.array_equal(got["times"], (np.arange(len(want)) / fps).astype(np.float32))
    assert np.abs(got["weights"].sum(1) - 1).max() <= 1e-6
    assert np.array_equal(got["faces"], np.asarray(faces).reshape(-1, 3))
    for n in got["gltf"]["skins"][0]["joints"]:
        q = got["keys"][n, "rotation"]
        assert (np.einsum("ki,ki->k", q[1:], q[:-1]) >= 0).all()          # sign continuity between keys
    return got


@pytest.fixture(autouse=True)
def _mat4(monkeypatch):
    """glb_check reads the vector accessor types; a skin's inverse bind matrices are MAT4 (16 components)."""
    monkeypatch.setitem(glb_check.NCOMP, "MAT4", 16)


# ---- the restatement's fits ------------------------------------------------------------------------------------------------
def test_piecewise_rigid_motion_is_recovered():
    """One FPS seed lands on each part, so n_bones = parts recovers every part's rigid motion to rounding."""
    v = rigid_parts()
    r = ref.fit(v, 4, 3)
    assert rms(v, r["history"][-1]) <= 1e-9
    assert sorted(np.unique(r["joints"][:, 0])) == [0, 1, 2, 3]


def test_smooth_skinning_is_approximated():
    """A 3-bone smooth skin: 8 bones reach at least 10x below the best single rigid transform (measured 2.0e-5x)."""
    v = bent_cylinder()
    one = ref.fit(v, 1, 5)["history"][-1]
    eight = ref.fit(v, 8, 5)["history"][-1]
    assert eight <= 0.1 * one
    assert eight <= 1e-4 * one


@pytest.mark.parametrize("n_bones", [3, 8])
def test_error_history_never_increases(n_bones):
    h = ref.fit(bent_cylinder(), n_bones, 6)["history"]
    assert all(b <= a for a, b in zip(h, h[1:])), h


def test_restated_kernels_keep_their_invariants():
    """Weights are non-negative, sum to 1 to rounding and use <= 4 distinct bones; rotations are proper and orthonormal."""
    v = bent_cylinder()
    r = ref.fit(v, 8, 3)
    w, j = r["weights"], r["joints"]
    assert (w >= 0).all() and np.abs(w.sum(1) - 1).max() <= 1e-12
    for row_j, row_w in zip(j, w):
        used = row_j[row_w > 0]
        assert len(set(used.tolist())) == len(used)
    R = r["transforms"][:, :, :9].reshape(-1, 3, 3)
    assert np.abs(R @ R.transpose(0, 2, 1) - np.eye(3)).max() <= 1e-12
    assert np.abs(np.linalg.det(R) - 1).max() <= 1e-12


def test_horn_rotation_of_degenerate_moments_is_identity():
    """A zero cross-covariance (one vertex, or points on a line through the centre) gives R = I."""
    R = ref.horn_rotation(np.zeros((1, 3, 3)))
    assert np.array_equal(R[0], np.eye(3).ravel())


# ---- the file ----------------------------------------------------------------------------------------------------------------
def _sphere_animation(frames=5):
    import standalone_tree as st

    sphere = st.textured_sphere()
    v = np.stack([sphere.vertices + 0.1 * t * np.sin(sphere.vertices * (t + 1)) for t in range(frames)])
    return sphere, v


def test_skinned_glb_round_trip(tmp_path):
    v = bent_cylinder()
    fit = as_fit(v, ref.fit(v, 8, 3))
    faces = np.random.default_rng(0).integers(0, v.shape[1], (50, 3))
    path = tmp_path / "skinned.glb"
    write_skinned_glb(path, fit, faces)
    got = check_skinned(path, fit, faces)
    assert got["gltf"]["materials"][0]["name"] == "BlueMaterial"
    assert np.abs(glb_check.blender_frame(reconstruct(fit)) - glb_check.blender_frame(v)).max() <= 0.05


def test_skinned_glb_keeps_the_visual(tmp_path):
    sphere, v = _sphere_animation()
    fit = as_fit(v, ref.fit(v, 6, 2))
    path = tmp_path / "skinned.glb"
    write_skinned_glb(path, fit, sphere.faces, fps=12, visual=sphere.visual)
    got = check_skinned(path, fit, sphere.faces, fps=12)
    prim = got["gltf"]["meshes"][0]["primitives"][0]
    uv = glb_check.accessor(got["gltf"], got["binary"], prim["attributes"]["TEXCOORD_0"])
    assert np.array_equal(uv, sphere.visual.uv)
    assert got["gltf"]["materials"][prim["material"]] == sphere.visual.material
    assert glb_check.image_bytes(got["gltf"], got["binary"]) == sphere.visual.image_bytes


def test_single_frame_and_single_bone(tmp_path):
    v = bent_cylinder(frames=1)
    fit = as_fit(v, ref.fit(v, 1, 1))
    path = tmp_path / "one.glb"
    write_skinned_glb(path, fit, [[0, 1, 2]])
    check_skinned(path, fit, [[0, 1, 2]])


# ---- argument checks ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape,n_bones,fill,match", [
    ((3, 10, 3), 2, np.nan, "non-finite"),
    ((3, 10, 3), 2, np.inf, "non-finite"),
    ((0, 10, 3), 2, 0.0, "T >= 1"),
    ((3, 10, 2), 2, 0.0, r"\(T, V, 3\)"),
    ((3, 10, 3), 0, 0.0, "n_bones"),
    ((3, 10, 3), 11, 0.0, "n_bones"),
    ((1, 300, 3), 257, 0.0, "n_bones"),
])
def test_fit_refuses_bad_arguments(shape, n_bones, fill, match):
    v = np.zeros(shape)
    if v.size:
        v.flat[0] = fill
    with pytest.raises(ValueError, match=match):
        fit_skinning(v, n_bones)


def test_writer_refuses_bad_fits(tmp_path):
    v = bent_cylinder(frames=2)
    fit = as_fit(v, ref.fit(v, 2, 1))
    with pytest.raises(ValueError, match="face"):
        write_skinned_glb(tmp_path / "a.glb", fit, np.zeros((0, 3), int))
    with pytest.raises(ValueError, match="outside"):
        write_skinned_glb(tmp_path / "a.glb", fit, [[0, 1, v.shape[1]]])
    fit.joints = fit.joints.copy()
    fit.joints[0, 0] = 2
    with pytest.raises(ValueError, match="joints"):
        write_skinned_glb(tmp_path / "a.glb", fit, [[0, 1, 2]])


# ---- the command line --------------------------------------------------------------------------------------------------------
def test_cli_flag_writes_the_skinned_glb(stubs, frames_dir, tmp_path, monkeypatch):
    """--skinning_bones N fits N bones to the animated GLB's vertices and writes skinned_mesh.glb; every other file is the
    same byte for byte as without the flag."""
    from actionmesh_b200 import inference, skinning

    calls = []

    def fake_fit(vertices, n_bones, device=None):
        calls.append((np.array(vertices), n_bones))
        return as_fit(vertices, ref.fit(vertices, n_bones, 1))

    monkeypatch.setattr(skinning, "fit_skinning", fake_fit)
    outs = [tmp_path / "plain", tmp_path / "skinned"]
    inference.main(["--input", str(frames_dir), "--output_dir", str(outs[0])])
    inference.main(["--input", str(frames_dir), "--output_dir", str(outs[1]), "--skinning_bones", "3"])
    names = sorted(p.name for p in outs[0].iterdir())
    assert sorted(p.name for p in outs[1].iterdir()) == sorted(names + ["skinned_mesh.glb"])
    for name in names:
        assert (outs[0] / name).read_bytes() == (outs[1] / name).read_bytes(), name
    assert len(calls) == 1 and calls[0][1] == 3
    anim = glb_check.read_animated(outs[1] / "animated_mesh.glb")
    fit = as_fit(calls[0][0], ref.fit(calls[0][0], 3, 1))
    check_skinned(outs[1] / "skinned_mesh.glb", fit, anim["faces"])
    assert inference.parse_args(["--input", "x"]).skinning_bones == 0


from test_inference_cpu import frames_dir, stubs  # noqa: E402,F401  (the command line's stubbed pipelines)
