"""The rig reader, the numpy restatement of the rig fit and the rig animation writer, on the CPU (DESIGN.md §21).

Files are built here by hand, and every check goes through `evaluate`, a numpy float64 statement of glTF skinning written
from the specification: node TRS -> world matrices -> sum_s w_s W_{j_s} IBM_{j_s} p for skinned primitives and W p for the
others."""
import json
import os
import struct
import subprocess

import numpy as np
import pytest

import glb_check
import rig_ref as ref
import skinning_ref
from actionmesh_b200 import gltf
from actionmesh_b200 import rig as rigmod

F32, U8, U16, U32 = 5126, 5121, 5123, 5125


@pytest.fixture(autouse=True)
def _mat4(monkeypatch):
    """glb_check reads the vector accessor types; a skin's inverse bind matrices are MAT4 (16 components)."""
    monkeypatch.setitem(glb_check.NCOMP, "MAT4", 16)


# ---- building files ------------------------------------------------------------------------------------------------------------
def axis_angle(axis, ang) -> np.ndarray:
    axis = np.asarray(axis, float) / np.linalg.norm(axis)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K @ K


def quat(m) -> np.ndarray:
    return gltf._quaternions(np.asarray(m))


def trs_matrix(t, q, s) -> np.ndarray:
    m = np.eye(4)
    m[:3, :3] = rigmod._rotation_matrix(q) * np.asarray(s, float)[None]
    m[:3, 3] = t
    return m


class Glb:
    """A minimal GLB writer for test files: buffer 0 is the BIN chunk."""

    def __init__(self):
        self.bin, self.views, self.accessors = bytearray(), [], []

    def acc(self, arr, comp, type_, normalized=False, min_max=False):
        arr = np.ascontiguousarray(arr, dtype={F32: "<f4", U8: "<u1", U16: "<u2", U32: "<u4"}[comp])
        self.bin += b"\0" * ((-len(self.bin)) % 4)
        self.views.append({"buffer": 0, "byteOffset": len(self.bin), "byteLength": arr.nbytes})
        self.bin += arr.tobytes()
        a = {"bufferView": len(self.views) - 1, "componentType": comp, "count": int(arr.shape[0]), "type": type_}
        if normalized:
            a["normalized"] = True
        if min_max:
            flat = arr.reshape(len(arr), -1)
            a["min"], a["max"] = flat.min(0).tolist(), flat.max(0).tolist()
        self.accessors.append(a)
        return len(self.accessors) - 1

    def write(self, path, doc):
        self.bin += b"\0" * ((-len(self.bin)) % 4)
        doc = {"asset": {"version": "2.0"}, **doc, "buffers": [{"byteLength": len(self.bin)}], "bufferViews": self.views,
               "accessors": self.accessors}
        js = json.dumps(doc).encode()
        js += b" " * ((-len(js)) % 4)
        body = struct.pack("<II", len(js), 0x4E4F534A) + js + struct.pack("<II", len(self.bin), 0x004E4942) + bytes(self.bin)
        with open(path, "wb") as f:
            f.write(b"glTF" + struct.pack("<II", 2, 12 + len(body)) + body)


# joint k: (parent, local translation); joint 3 (the neck, intermediate) and joint 10 (a leaf) influence nothing
SKELETON = [(-1, [0.1, 0.2, 0.0]), (0, [0, 1, 0]), (1, [0, 1, 0]), (2, [0, .8, 0]), (3, [0, .5, 0]), (2, [.6, .3, 0]),
            (5, [.8, 0, 0]), (2, [-.6, .3, 0]), (7, [-.8, 0, 0]), (0, [.3, -.2, 0]), (9, [0, -1, 0])]
LIVE = [0, 1, 2, 4, 5, 6, 7, 8, 9]
TIP = {0: 1, 1: 2, 2: 3, 3: 4, 4: None, 5: 6, 6: None, 7: 8, 8: None, 9: 10}


def rigged_file(path, V=300, seed=0, *, skin_order=None, matrix_joint=4, two_prims=True, rigid=True, static=True,
                armature=True, live=LIVE, mutate=None):
    """A Mixamo-like file: an "Armature" node (90 degrees about X, scale 0.01) above the root joint and the skinned mesh
    node; the skin's joints in `skin_order` (a permutation of SKELETON); joint `matrix_joint` stored as `matrix`; two
    skinned primitives with different materials (u8 joints + float weights; u16 joints + normalized u16 / u8 weights in two
    sets); a rigid child mesh under joint 6 and a static mesh at the scene root.  `mutate(doc, glb)` edits the JSON before
    writing.  -> the JSON."""
    rng = np.random.default_rng(seed)
    J = len(SKELETON)
    skin_order = list(range(J)) if skin_order is None else list(skin_order)
    q0 = quat(np.stack([axis_angle(rng.standard_normal(3), rng.uniform(0, .3)) for _ in range(J)]))
    scale = np.ones((J, 3))
    scale[4] = 1.2
    arm = trs_matrix([0.5, 0, 0.2], quat(axis_angle([1, 0, 0], np.pi / 2)), [0.01] * 3) if armature else np.eye(4)
    mesh_local = trs_matrix([0.0, 0.1, 0.0], [0, 0, 0, 1], [1, 1, 1])
    G0 = np.zeros((J, 4, 4))
    for j, (p, t) in enumerate(SKELETON):
        G0[j] = (G0[p] if p >= 0 else arm) @ trs_matrix(t, q0[j], scale[j])
    mesh_world = arm @ mesh_local
    heads = G0[:, :3, 3]
    pick = rng.choice(live, V)
    tip = np.array([heads[TIP[j]] if TIP[j] is not None else heads[j] + 0.5 * (heads[j] - heads[SKELETON[j][0]])
                    for j in pick])
    world_pts = heads[pick] + rng.uniform(0, 1, (V, 1)) * (tip - heads[pick]) + 0.0008 * rng.standard_normal((V, 3))
    inv_mesh = np.linalg.inv(mesh_world)
    local_pts = world_pts @ inv_mesh[:3, :3].T + inv_mesh[:3, 3]
    jnt = np.zeros((V, 8), np.int64)
    wgt = np.zeros((V, 8))
    for i in range(V):
        j = pick[i]
        js = [j] + ([SKELETON[j][0]] if SKELETON[j][0] >= 0 and i % 3 else [])
        js += [TIP[j]] if i % 3 == 2 and TIP[j] is not None and TIP[j] in live else []
        w = rng.uniform(0.2, 1, len(js))
        slots = [0, 5, 2][:len(js)] if i % 2 else list(range(len(js)))         # used slots in either set
        jnt[i, slots], wgt[i, slots] = js, w / w.sum()
    # the file's joint index of skeleton joint j
    file_index = {j: skin_order.index(j) for j in range(J)}
    jnt_file = np.vectorize(file_index.get)(jnt)
    g = Glb()
    node_of = {j: 1 + k for k, j in enumerate(skin_order)}           # node 1 + k holds skin joint k
    nodes = [{"name": "Armature", "children": [node_of[0]]}]
    nodes[0].update(**({"rotation": quat(axis_angle([1, 0, 0], np.pi / 2)).tolist(), "scale": [0.01] * 3,
                        "translation": [0.5, 0, 0.2]} if armature else {}))
    for j in skin_order:
        nd = {"name": f"J{j}"}
        if j == matrix_joint:
            nd["matrix"] = trs_matrix(SKELETON[j][1], q0[j], scale[j]).T.ravel().tolist()
        else:
            nd.update(translation=list(map(float, SKELETON[j][1])), rotation=q0[j].tolist(), scale=scale[j].tolist())
        kids = [node_of[c] for c in range(J) if SKELETON[c][0] == j]
        if kids:
            nd["children"] = kids
        nodes.append(nd)
    half = V // 2 if two_prims else V
    prims = []
    for lo, hi, big in ((0, half, False), (half, V, True))[:2 if two_prims else 1]:
        idx = np.arange(hi - lo)
        faces = np.stack([idx[:-2], idx[1:-1], idx[2:]], 1)
        attrs = {"POSITION": g.acc(local_pts[lo:hi], F32, "VEC3", min_max=True)}
        if big:
            attrs["JOINTS_0"] = g.acc(jnt_file[lo:hi, :4], U16, "VEC4")
            attrs["JOINTS_1"] = g.acc(jnt_file[lo:hi, 4:], U16, "VEC4")
            attrs["WEIGHTS_0"] = g.acc(np.round(wgt[lo:hi, :4] * 65535), U16, "VEC4", normalized=True)
            attrs["WEIGHTS_1"] = g.acc(np.round(wgt[lo:hi, 4:] * 255), U8, "VEC4", normalized=True)
        else:
            # one set: fold slots 4..7 into 0..3 (their joints differ from slot 0's only where used)
            j4, w4 = jnt_file[lo:hi].copy(), wgt[lo:hi].copy()
            mv = w4[:, 5] > 0
            j4[mv, 1], w4[mv, 1] = j4[mv, 5], w4[mv, 5]
            attrs["JOINTS_0"] = g.acc(j4[:, :4], U8, "VEC4")
            attrs["WEIGHTS_0"] = g.acc(w4[:, :4], F32, "VEC4")
        prims.append({"attributes": attrs, "indices": g.acc(faces.reshape(-1, 1), U32, "SCALAR"), "material": len(prims)})
    meshes = [{"primitives": prims}]
    nodes.append({"name": "Body", "mesh": 0, "skin": 0, "translation": [0.0, 0.1, 0.0]})
    nodes[0]["children"].append(len(nodes) - 1)
    box = np.array([[0, 0, 0], [.1, 0, 0], [0, .1, 0], [0, 0, .1]], float)
    tri = np.array([[0, 1, 2], [0, 2, 3], [0, 3, 1], [1, 3, 2]])
    if rigid:
        meshes.append({"primitives": [{"attributes": {"POSITION": g.acc(box, F32, "VEC3", min_max=True)},
                                       "indices": g.acc(tri.reshape(-1, 1), U32, "SCALAR")}]})
        nodes.append({"name": "Prop", "mesh": len(meshes) - 1, "translation": [0.4, 0.1, 0.0], "rotation":
                      quat(axis_angle([0, 0, 1], 0.4)).tolist()})
        nodes[node_of[6]].setdefault("children", []).append(len(nodes) - 1)
    roots = [0]
    if static:
        meshes.append({"primitives": [{"attributes": {"POSITION": g.acc(box + 3, F32, "VEC3", min_max=True)},
                                       "indices": g.acc(tri.reshape(-1, 1), U32, "SCALAR")}]})
        nodes.append({"name": "Ground", "mesh": len(meshes) - 1})
        roots.append(len(nodes) - 1)
    ibm = np.stack([np.linalg.inv(G0[j]) @ mesh_world for j in skin_order])
    doc = {"scene": 0, "scenes": [{"nodes": roots}], "nodes": nodes, "meshes": meshes,
           "materials": [{"name": "A"}, {"name": "B"}],
           "skins": [{"joints": [node_of[j] for j in skin_order], "skeleton": node_of[0],
                      "inverseBindMatrices": g.acc(ibm.transpose(0, 2, 1).reshape(J, 16), F32, "MAT4")}],
           "animations": [{"name": "Idle", "channels": [{"sampler": 0, "target": {"node": node_of[1], "path": "rotation"}}],
                           "samplers": [{"input": g.acc(np.array([[0.0], [1.0]]), F32, "SCALAR", min_max=True),
                                         "output": g.acc(np.tile(q0[1], (2, 1)), F32, "VEC4")}]}]}
    if mutate is not None:
        mutate(doc, g)
    g.write(path, doc)
    return doc


# ---- the independent evaluator -------------------------------------------------------------------------------------------------
def read_file(path):
    data = open(path, "rb").read()
    jlen = struct.unpack_from("<I", data, 12)[0]
    doc = json.loads(data[20:20 + jlen])
    return doc, data[28 + jlen:]


def evaluate(path, key=None) -> np.ndarray:
    """(V, 3) of the file at `path` in load_glb's vertex order: the default pose, or key `key` of animations[0]."""
    doc, binary = read_file(path)
    acc = lambda i: glb_check.accessor(doc, binary, i).astype(np.float64)
    nodes = doc["nodes"]
    local = {}
    for n, nd in enumerate(nodes):
        if "matrix" in nd:
            local[n] = np.asarray(nd["matrix"], float).reshape(4, 4).T
        else:
            local[n] = [np.asarray(nd.get("translation", [0, 0, 0]), float), np.asarray(nd.get("rotation", [0, 0, 0, 1]), float),
                        np.asarray(nd.get("scale", [1, 1, 1]), float)]
    if key is not None:
        anim = doc["animations"][0]
        for ch in anim["channels"]:
            n, p = ch["target"]["node"], ch["target"]["path"]
            v = acc(anim["samplers"][ch["sampler"]]["output"])[key]
            local[n][{"translation": 0, "rotation": 1, "scale": 2}[p]] = v
    mat = {}
    for n, l in local.items():
        if isinstance(l, list):
            x, y, z, w = l[1] / np.linalg.norm(l[1])
            r = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                          [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                          [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
            m = np.eye(4)
            m[:3, :3] = r * l[2][None]
            m[:3, 3] = l[0]
            mat[n] = m
        else:
            mat[n] = l
    world, order = {}, []

    def visit(n, parent):
        world[n] = parent @ mat[n]
        order.append(n)
        for c in nodes[n].get("children", []):
            visit(c, world[n])

    for r in doc["scenes"][doc.get("scene", 0)]["nodes"]:
        visit(r, np.eye(4))
    out = []
    for n in order:
        if "mesh" not in nodes[n]:
            continue
        for prim in doc["meshes"][nodes[n]["mesh"]]["primitives"]:
            p = acc(prim["attributes"]["POSITION"])
            if "skin" in nodes[n]:
                skin = doc["skins"][nodes[n]["skin"]]
                ibm = acc(skin["inverseBindMatrices"]).reshape(-1, 4, 4).transpose(0, 2, 1)
                jm = np.stack([world[j] for j in skin["joints"]]) @ ibm
                a = prim["attributes"]
                js = np.concatenate([glb_check.accessor(doc, binary, a[k]) for k in ("JOINTS_0", "JOINTS_1") if k in a], 1)
                ws = []
                for k in ("WEIGHTS_0", "WEIGHTS_1"):
                    if k in a:
                        w = acc(a[k])
                        if doc["accessors"][a[k]].get("normalized"):
                            w = w / np.iinfo(glb_check.DTYPES[doc["accessors"][a[k]]["componentType"]]).max
                        ws.append(w)
                ws = np.concatenate(ws, 1)
                ws = ws / ws.sum(1, keepdims=True)
                v = np.zeros_like(p)
                for s in range(js.shape[1]):
                    m = jm[js[:, s].astype(np.int64)]
                    v += ws[:, s:s + 1] * (np.einsum("vij,vj->vi", m[:, :3, :3], p) + m[:, :3, 3])
                out.append(v)
            else:
                out.append(p @ world[n][:3, :3].T + world[n][:3, 3])
    return np.concatenate(out)


def animation(rig, T, seed=1, max_deg=60.0):
    """Local rotation matrices (T, J, 9) and translations (T, J, 3) in topological order: every joint's default rotation
    times a random rotation of up to max_deg degrees, and a moving root."""
    a = rigmod.rig_arrays(rig)
    rng = np.random.default_rng(seed)
    J = len(a.parent)
    rots = np.zeros((T, J, 9))
    trs = np.ascontiguousarray(np.broadcast_to(a.translations, (T, J, 3)))
    for t in range(T):
        for j in range(J):
            rots[t, j] = (a.rotations[j].reshape(3, 3)
                          @ axis_angle(rng.standard_normal(3), np.deg2rad(rng.uniform(0, max_deg)))).ravel()
        for j in np.flatnonzero(a.parent < 0):
            trs[t, j] = a.translations[j] + 0.5 * rng.standard_normal(3)
    return a, rots, trs


def fit_of(a, rots, trs) -> rigmod.RigFit:
    """A RigFit holding the topological-order state (rots, trs), joints back in skin order."""
    T, J = rots.shape[:2]
    m = np.empty_like(rots)
    m[:, a.order] = rots
    t = np.empty_like(trs)
    t[:, a.order] = trs
    m = m.reshape(T, J, 3, 3)
    return rigmod.RigFit(rotations=gltf._quaternions(m), rotation_matrices=m, translations=t, history=[], rms_error=0.0,
                         max_error=0.0)


# ---- reading ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("skin_order", [None, [4, 0, 1, 2, 3, 10, 5, 6, 7, 8, 9]])
def test_load_rig_reads_the_file(tmp_path, skin_order):
    path = tmp_path / "rigged.glb"
    rigged_file(path, skin_order=skin_order)
    rig = gltf.load_rig(path)
    mesh = gltf.load_glb(path)
    assert np.array_equal(rig.rest.view(np.uint64), mesh.vertices.view(np.uint64))   # bit for bit
    J = len(SKELETON)
    order = list(range(J)) if skin_order is None else skin_order
    assert [rig.parent[k] for k in range(J)] == [order.index(SKELETON[j][0]) if SKELETON[j][0] >= 0 else -1 for j in order]
    pos = {int(j): k for k, j in enumerate(rig.order)}
    assert all(pos[int(rig.parent[j])] < pos[j] for j in range(J) if rig.parent[j] >= 0)
    assert rig.from_matrix.tolist() == [j == 4 for j in order]
    V = len(rig.rest)
    # the rigid child under joint 6 comes first (depth-first order), the static box last
    assert (rig.slot_weight[:4, 0] == 1).all() and (rig.slot_bind[:4, 0] == J).all() and len(rig.binds) == J + 1
    assert rig.joint_nodes[rig.bind_joint[J]] == 1 + order.index(6)
    assert np.allclose(rig.slot_weight.sum(1)[:-4], 1.0) and (rig.slot_weight[-4:] == 0).all()
    assert (np.diff((rig.slot_weight > 0).astype(int), axis=1) <= 0).all()                      # used slots first
    # the rig's pose of random joint rotations equals glTF skinning of the same TRS
    a, rots, trs = animation(rig, 2, max_deg=60)
    want = ref.posed(a, rots, trs)
    for t in range(2):
        doc, _ = read_file(path)
        fit = fit_of(a, rots, trs)
        out = tmp_path / f"posed{t}.glb"
        gltf.write_rig_animation(path, out, rig, fit)
        got = evaluate(out, key=t)
        assert np.abs(got - want[t]).max() <= 1e-5 * np.abs(want).max(), t
    assert V == len(mesh.vertices)


def test_default_pose_is_the_rest(tmp_path):
    path = tmp_path / "rigged.glb"
    rigged_file(path)
    rig = gltf.load_rig(path)
    a = rigmod.rig_arrays(rig)
    posed = ref.posed(a, a.rotations[None], a.translations[None])[0]
    diag = np.linalg.norm(rig.rest.max(0) - rig.rest.min(0))
    assert np.abs(posed - rig.rest).max() <= 1e-9 * diag
    assert np.abs(evaluate(path) - rig.rest).max() <= 1e-6 * diag


def _refused(tmp_path, match, **kw):
    path = tmp_path / "bad.glb"
    rigged_file(path, **kw)
    with pytest.raises(ValueError, match=match):
        gltf.load_rig(path)


def _skin_attr(doc, name, value):
    doc["meshes"][0]["primitives"][1]["attributes"][name] = value


def test_refusals(tmp_path):
    def no_skin(doc, g):
        for nd in doc["nodes"]:
            nd.pop("skin", None)

    _refused(tmp_path, "no included mesh node has a skin", mutate=no_skin)

    def two_skins(doc, g):
        doc["skins"].append(dict(doc["skins"][0]))
        doc["nodes"].append({"mesh": 0, "skin": 1})
        doc["scenes"][0]["nodes"].append(len(doc["nodes"]) - 1)

    _refused(tmp_path, "2 distinct skins", mutate=two_skins)

    def instanced(doc, g):
        doc["nodes"].append({"mesh": 0})
        doc["scenes"][0]["nodes"].append(len(doc["nodes"]) - 1)

    _refused(tmp_path, "instanced by 2 nodes", mutate=instanced)

    def nine(doc, g):
        _skin_attr(doc, "JOINTS_2", doc["meshes"][0]["primitives"][1]["attributes"]["JOINTS_0"])
        _skin_attr(doc, "WEIGHTS_2", doc["meshes"][0]["primitives"][1]["attributes"]["WEIGHTS_0"])

    _refused(tmp_path, "more than 8 influences", mutate=nine)

    def zero_row(doc, g):
        n = g.accessors[doc["meshes"][0]["primitives"][0]["attributes"]["POSITION"]]["count"]
        doc["meshes"][0]["primitives"][0]["attributes"]["WEIGHTS_0"] = g.acc(np.zeros((n, 4)), F32, "VEC4")

    _refused(tmp_path, "sum to 0", mutate=zero_row)

    def outside(doc, g):
        n = g.accessors[doc["meshes"][0]["primitives"][0]["attributes"]["POSITION"]]["count"]
        doc["meshes"][0]["primitives"][0]["attributes"]["JOINTS_0"] = g.acc(np.full((n, 4), 40), U8, "VEC4")

    _refused(tmp_path, "outside the skin", mutate=outside)

    def sheared_parent(doc, g):
        doc["nodes"][0]["scale"] = [0.01, 0.02, 0.01]

    _refused(tmp_path, "not a rotation times a positive uniform scale", mutate=sheared_parent)

    def shear(doc, g):
        m = np.asarray(doc["nodes"][5]["matrix"]).reshape(4, 4).T
        m[0, 1] += 0.3
        doc["nodes"][5]["matrix"] = m.T.ravel().tolist()

    _refused(tmp_path, "shear", mutate=shear)

    def negative(doc, g):
        m = np.asarray(doc["nodes"][5]["matrix"]).reshape(4, 4).T
        m[:3, 0] *= -1
        doc["nodes"][5]["matrix"] = m.T.ravel().tolist()

    _refused(tmp_path, "non-positive scale", mutate=negative)

    def morph(doc, g):
        prim = doc["meshes"][0]["primitives"][0]
        prim["targets"] = [{"POSITION": prim["attributes"]["POSITION"]}]
        doc["meshes"][0]["weights"] = [0.5]

    _refused(tmp_path, "morph targets with non-zero", mutate=morph)

    def moved(doc, g):
        doc["nodes"][-3]["translation"] = [0.0, 5.0, 0.0]

    _refused(tmp_path, "not the bind pose", mutate=moved)


def test_refuses_an_external_buffer(tmp_path):
    path = tmp_path / "ext.glb"
    rigged_file(path)
    doc, binary = read_file(path)
    doc["buffers"].append({"uri": "other.bin", "byteLength": 4})
    js = json.dumps(doc).encode()
    js += b" " * ((-len(js)) % 4)
    body = struct.pack("<II", len(js), 0x4E4F534A) + js + struct.pack("<II", len(binary), 0x004E4942) + binary
    path.write_bytes(b"glTF" + struct.pack("<II", 2, 12 + len(body)) + body)
    with pytest.raises(ValueError, match="external file"):
        gltf.load_rig(path)
    # no BIN chunk: buffer 0 as a data URI
    import base64

    doc["buffers"] = [{"uri": "data:application/octet-stream;base64," + base64.b64encode(binary).decode(),
                       "byteLength": len(binary)}]
    js = json.dumps(doc).encode()
    js += b" " * ((-len(js)) % 4)
    body = struct.pack("<II", len(js), 0x4E4F534A) + js
    path.write_bytes(b"glTF" + struct.pack("<II", 2, 12 + len(body)) + body)
    with pytest.raises(ValueError, match="BIN chunk"):
        gltf.load_rig(path)


def test_morph_targets_with_zero_weights_are_accepted(tmp_path):
    def morph(doc, g):
        prim = doc["meshes"][0]["primitives"][0]
        prim["targets"] = [{"POSITION": prim["attributes"]["POSITION"]}]
        doc["meshes"][0]["weights"] = [0.0]

    path = tmp_path / "m.glb"
    rigged_file(path, mutate=morph)
    gltf.load_rig(path)


# ---- the restatement ---------------------------------------------------------------------------------------------------------
def _exact_animation(tmp_path, V=240, T=2):
    path = tmp_path / "rigged.glb"
    rigged_file(path, V=V)
    rig = gltf.load_rig(path)
    a, rots, trs = animation(rig, T)
    return path, rig, a, rots, trs, ref.posed(a, rots, trs)


def synthetic_rig(V=400, T=3, seed=0):
    """An exact FK animation of an 11-joint branching rig of depth 5 under an armature transform (scale 0.01, 90 degrees
    about X): every joint but one leaf has vertices in a cloud around its bone (radius 8 bone lengths: thin limbs converge far slower, DESIGN §21), weighted to it, its
    parent and its child; every local rotation is turned by up to 60 degrees in every frame and the root moves.
    -> (RigArrays, vertices (T, V, 3))."""
    from types import SimpleNamespace

    rng = np.random.default_rng(seed)
    J = len(SKELETON)
    parent = np.array([p for p, _ in SKELETON])
    trans = np.array([t for _, t in SKELETON], float)
    q0 = quat(np.stack([axis_angle(rng.standard_normal(3), rng.uniform(0, .3)) for _ in range(J)]))
    scale = np.ones((J, 3))
    scale[4] = 1.2
    above = np.tile(np.eye(4), (J, 1, 1))
    above[0] = trs_matrix([0.5, 0, 0.2], quat(axis_angle([1, 0, 0], np.pi / 2)), [0.01] * 3)
    G0 = np.zeros((J, 4, 4))
    for j in range(J):
        G0[j] = (G0[parent[j]] if parent[j] >= 0 else above[j]) @ trs_matrix(trans[j], q0[j], scale[j])
    heads = G0[:, :3, 3]
    pick = rng.choice(list(range(10)), V)
    tip = np.array([heads[TIP[j]] if TIP[j] is not None else heads[j] + 0.5 * (heads[j] - heads[parent[j]]) for j in pick])
    pts = heads[pick] + rng.uniform(0, 1, (V, 1)) * (tip - heads[pick]) + 0.08 * rng.standard_normal((V, 3))
    sb, sw = np.zeros((V, 8), np.int32), np.zeros((V, 8))
    for i in range(V):
        j = pick[i]
        js = [j] + ([parent[j]] if parent[j] >= 0 and i % 3 else []) + ([TIP[j]] if i % 3 == 2 and TIP[j] else [])
        w = rng.uniform(0.2, 1, len(js))
        sb[i, :len(js)], sw[i, :len(js)] = js, w / w.sum()
    rig = SimpleNamespace(order=np.arange(J), parent=parent, scale=scale, above=above, binds=np.linalg.inv(G0),
                          bind_joint=np.arange(J), rotation=q0, translation=trans, points=pts, rest=pts.copy(),
                          slot_bind=sb, slot_weight=sw)
    a, rots, trs = animation(rig, T, seed=seed + 1)
    return rig, a, ref.posed(a, rots, trs)


def test_restatement_recovers_an_exact_animation():
    """The default sweeps reach 1e-6 of the diagonal on `synthetic_rig`, and the error never increases beyond rounding."""
    _, a, verts = synthetic_rig()
    rot, trans, history = ref.fit(a, verts, rigmod.DEFAULT_SWEEPS)
    T, V = verts.shape[:2]
    diag = np.linalg.norm(a.rest.max(0) - a.rest.min(0))
    rms = np.sqrt(history[-1] / (T * V)) / diag
    assert rms <= 1e-6, rms
    assert all(b <= a_ * (1 + 1e-12) + 1e-30 for a_, b in zip(history, history[1:])), history


def test_one_joint_fit_is_the_rigid_horn_fit():
    """One root joint, every vertex on it with weight 1, identity above and binds: the rotation update is skinning_ref's
    rigid Horn fit about the joint's origin."""
    rng = np.random.default_rng(3)
    V, T = 500, 3
    p = rng.standard_normal((V, 3))
    verts = np.stack([p @ axis_angle(rng.standard_normal(3), 0.7).T + rng.standard_normal(3) for _ in range(T)])
    a = rigmod.RigArrays(order=np.array([0]), parent=np.array([-1], np.int32), subtree_end=np.array([1]),
                         scale=np.ones((1, 3)), above=rigmod._xf12(np.eye(4)[None]), above_inv=np.eye(3).reshape(1, 9),
                         binds=rigmod._xf12(np.eye(4)[None]), bind_joint=np.array([0], np.int32),
                         rotations=np.eye(3).reshape(1, 9), translations=np.zeros((1, 3)), points=p, rest=p,
                         slot_bind=np.zeros((V, 8), np.int32), slot_weight=np.pad(np.ones((V, 1)), ((0, 0), (0, 7))),
                         lists=np.arange(V, dtype=np.int32), offsets=np.array([0, V]))
    rot = np.tile(np.eye(3).reshape(1, 1, 9), (T, 1, 1))
    trans = np.zeros((T, 1, 3))
    got = ref.rotation_update(a, rot, trans, verts, a.lists, 0, 1)
    # skinning_ref's Horn fit of the same cross-covariance H = sum p v^T (no centring: the pivot is the origin)
    for t in range(T):
        H = (p[:, :, None] * verts[t][:, None, :]).reshape(-1, 9)
        Hs = skinning_ref.sum_in_order(skinning_ref.tile_partials(H)).reshape(1, 3, 3)
        want = skinning_ref.horn_rotation(Hs)[0]
        assert np.abs(got[t, 0] - want).max() <= 1e-12
    # and the translation update then moves the root to the residual's mean
    tr = ref.translation_update(a, got, trans, verts, a.lists, 0, 1)
    res = verts - np.einsum("tij,vj->tvi", got[:, 0].reshape(T, 3, 3), p)
    assert np.abs(tr[:, 0] - res.mean(1)).max() <= 1e-12


# ---- the writer --------------------------------------------------------------------------------------------------------------
def test_writer_keeps_the_file_and_adds_one_animation(tmp_path):
    path, rig, a, rots, trs, verts = _exact_animation(tmp_path, V=120, T=3)
    fit = fit_of(a, rots, trs)
    out = tmp_path / "rigged_mesh.glb"
    gltf.write_rig_animation(path, out, rig, fit, fps=8)
    glb_check.check_glb(out)
    src, src_bin = read_file(path)
    doc, binary = read_file(out)
    assert binary[:len(src_bin)] == src_bin
    for key in ("scenes", "meshes", "skins", "materials"):
        assert doc[key] == src[key], key
    for n, (x, y) in enumerate(zip(src["nodes"], doc["nodes"])):
        if "matrix" in x:
            j = rig.joint_nodes.index(n)
            assert {k: v for k, v in x.items() if k != "matrix"} == {k: v for k, v in y.items()
                                                                     if k not in ("translation", "rotation", "scale")}
            assert np.allclose(trs_matrix(y["translation"], y["rotation"], y["scale"]),
                               np.asarray(x["matrix"]).reshape(4, 4).T, atol=1e-12), j
        else:
            assert x == y
    assert doc["accessors"][:len(src["accessors"])] == src["accessors"]
    assert doc["bufferViews"][:len(src["bufferViews"])] == src["bufferViews"]
    assert doc["animations"][1:] == src["animations"]
    anim = doc["animations"][0]
    assert anim["name"] == "ActionMesh"
    paths = sorted((c["target"]["node"], c["target"]["path"]) for c in anim["channels"])
    roots = [rig.joint_nodes[j] for j in range(len(rig.joint_nodes)) if rig.parent[j] < 0]
    assert paths == sorted([(n, "rotation") for n in rig.joint_nodes] + [(n, "translation") for n in roots])
    for s in anim["samplers"]:
        assert s["interpolation"] == "LINEAR"
        times = glb_check.accessor(doc, binary, s["input"])[:, 0]
        assert np.array_equal(times, (np.arange(3) / 8).astype(np.float32))
    for c in anim["channels"]:
        if c["target"]["path"] == "rotation":
            q = glb_check.accessor(doc, binary, anim["samplers"][c["sampler"]]["output"]).astype(np.float64)
            assert (np.einsum("ki,ki->k", q[1:], q[:-1]) >= 0).all()
    for t in range(3):
        got = evaluate(out, key=t)
        assert np.abs(got - verts[t]).max() <= 2.0 ** -18 * max(1.0, np.abs(verts).max()), t


def test_write_refuses_a_mismatched_fit(tmp_path):
    path, rig, a, rots, trs, _ = _exact_animation(tmp_path, V=60, T=2)
    fit = fit_of(a, rots, trs)
    fit.rotations = fit.rotations[:, :-1]
    with pytest.raises(ValueError, match="do not match"):
        gltf.write_rig_animation(path, tmp_path / "o.glb", rig, fit)


# ---- the command line --------------------------------------------------------------------------------------------------------
def test_cli_keep_rig_needs_a_rigged_mesh_input(tmp_path, capsys):
    from actionmesh_b200 import inference

    with pytest.raises(SystemExit):
        inference.parse_args(["--input", "x.mp4", "--keep_rig"])
    assert "--keep_rig needs --mesh_input" in capsys.readouterr().err
    plain = tmp_path / "plain.glb"
    rigged_file(plain, mutate=lambda doc, g: [nd.pop("skin", None) for nd in doc["nodes"]])
    with pytest.raises(SystemExit, match="no included mesh node has a skin"):
        inference.main(["--input", "x.mp4", "--mesh_input", str(plain), "--keep_rig", "--weights_root",
                        str(tmp_path / "missing")])


def test_cli_flag_writes_the_rigged_glb(tmp_path, monkeypatch):
    """run_actionmesh with a rig: the fit sees the animated GLB's (T, V, 3) vertices and rigged_mesh.glb is written;
    without it nothing changes."""
    from actionmesh_b200 import inference
    from actionmesh_b200.pipeline import Mesh

    path = tmp_path / "rigged.glb"
    rigged_file(path, V=60)
    rig = gltf.load_rig(path)
    a, rots, trs = animation(rig, 3)
    verts = ref.posed(a, rots, trs)
    seen = {}

    class Pipe:
        device = "cpu"

        def __call__(self, input, anchor_mesh, seed, **kw):
            return [Mesh(vertices=v, faces=np.asarray(anchor_mesh.faces)) for v in verts]

    def fake_fit(r, vertices, device=None):
        seen["v"] = vertices
        return fit_of(a, rots, trs)

    monkeypatch.setattr(inference, "load_frames", lambda *a_, **k: type("F", (), {"frames": []})())
    monkeypatch.setattr(inference.rig_fit, "fit_rig_animation", fake_fit)
    monkeypatch.setattr(inference.render, "B200MeshVisualizer", lambda **k: type("V", (), {"render": lambda *a_, **k_: None})())
    outs = [tmp_path / "plain", tmp_path / "rig"]
    inference.run_actionmesh(Pipe(), "x", str(outs[0]), mesh_input=str(path))
    inference.run_actionmesh(Pipe(), "x", str(outs[1]), mesh_input=str(path), rig=rig)
    names = sorted(p.name for p in outs[0].iterdir())
    assert sorted(p.name for p in outs[1].iterdir()) == sorted(names + ["rigged_mesh.glb"])
    for name in names:
        assert (outs[0] / name).read_bytes() == (outs[1] / name).read_bytes(), name
    assert np.array_equal(seen["v"], verts)
    assert np.abs(evaluate(outs[1] / "rigged_mesh.glb", key=2) - verts[2]).max() <= 1e-5


# ---- the kernels compile without spills -----------------------------------------------------------------------------------------
def test_rig_kernels_do_not_spill(tmp_path):
    import re

    import __graft_entry__ as ge

    obj = str(tmp_path / "rig.o")
    res = subprocess.run([ge._nvcc(), *ge.NVCC_FLAGS, "-c", os.path.join(ge.CSRC, "rig.cu"), "-o", obj],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    entries = re.findall(r"Function properties for (\w+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads", res.stdout + res.stderr)
    rig_kernels = [e for e in entries if "rig_" in e[0]]
    assert len(rig_kernels) >= 6
    for name, _, stores, loads in rig_kernels:
        assert stores == "0" and loads == "0", f"{name} spills {stores} B / loads {loads} B"
