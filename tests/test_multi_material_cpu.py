"""Multi-primitive inputs keep every material (no GPU): `gltf.load_glb` reads a `GltfMultiVisual` from hand-built files,
the three writers give each primitive back its range and material, the texture modality builds one shading record per
(material, has UVs) pair, and the command line hands the visual to both writers and to the renderer."""
import io
import logging

import numpy as np
import pytest
import torch
from PIL import Image
from scipy.spatial.transform import Rotation

import glb_check
import skinning_ref as sref
from actionmesh_b200 import ops, render
from actionmesh_b200.gltf import (ANIMATED_GLB_MAP, DEFAULT_MATERIAL, GltfMultiVisual, GltfVisual, load_glb,
                                  write_animated_glb, write_glb, write_skinned_glb)
from actionmesh_b200.pipeline import Mesh
from test_gltf_cpu import Glb
from test_skinning_cpu import _mat4, as_fit  # noqa: F401  (_mat4: glb_check reads the skin's MAT4 accessor)

f32 = np.float32


def png(img: np.ndarray) -> bytes:
    buf = io.BytesIO()
    Image.fromarray(img).save(buf, format="PNG")
    return buf.getvalue()


def split(vertices, faces, uv, groups):
    """A mesh re-laid out as primitives: group p's faces (indices into `faces`) get their own copies of the vertices they
    use -> (vertices, faces, uv, vertex_ranges, face_ranges), the layout `load_glb` reads."""
    vs, fs, uvs, vr, fr, n = [], [], [], [], [], 0
    faces = np.asarray(faces)
    for g in groups:
        used, local = np.unique(faces[g], return_inverse=True)
        vs.append(np.asarray(vertices)[used])
        uvs.append(np.asarray(uv)[used])
        fs.append(local.reshape(-1, 3) + n)
        vr.append((n, len(used)))
        fr.append((sum(c for _, c in fr), len(g)))
        n += len(used)
    return (np.concatenate(vs), np.concatenate(fs).astype(np.int64), np.concatenate(uvs).astype(f32),
            np.array(vr, np.int64), np.array(fr, np.int64))


# ---- a hand-built file ------------------------------------------------------------------------------------------------------
def _node(t, q, s):
    return {"translation": list(t), "rotation": list(q), "scale": list(s)}


def _world(node):
    m = np.eye(4)
    m[:3, :3] = Rotation.from_quat(node["rotation"]).as_matrix() @ np.diag(node["scale"])
    m[:3, 3] = node["translation"]
    return m


@pytest.fixture
def built(tmp_path):
    """Mesh A: a textured triangle pair (material 0) and a UV-less strip (material 1); mesh B: points, a textured
    material-less primitive and a factor-only one (material 2).  Materials 0 and 1 use two textures of one image and one
    sampler.  Node 0 places A, node 1 mirrors B, node 2 places A again -> (path, expected)."""
    rng = np.random.default_rng(7)
    g = Glb()
    a0v, a0uv, a0f = rng.standard_normal((4, 3)).astype(f32), rng.random((4, 2)).astype(f32), np.array([[0, 1, 2], [0, 2, 3]])
    a1v, strip = rng.standard_normal((5, 3)).astype(f32), np.array([0, 1, 2, 3, 4])
    b1v, b1uv, b1f = rng.standard_normal((3, 3)).astype(f32), rng.random((3, 2)).astype(f32), np.array([[0, 1, 2]])
    b2v, b2uv, b2f = rng.standard_normal((6, 3)).astype(f32), rng.random((6, 2)).astype(f32), np.array([[0, 1, 2], [3, 4, 5], [1, 3, 5]])
    img = png(rng.integers(0, 255, (4, 6, 3), dtype=np.uint8))
    image_view = g.view(img)
    prims_a = [{"attributes": {"POSITION": g.positions(a0v), "TEXCOORD_0": g.accessor(a0uv, 5126, "VEC2")},
                "indices": g.indices(a0f, 5123), "material": 0},
               {"attributes": {"POSITION": g.positions(a1v)}, "indices": g.indices(strip, 5121), "mode": 5, "material": 1}]
    prims_b = [{"attributes": {"POSITION": g.positions(b1v)}, "mode": 0, "material": 1},
               {"attributes": {"POSITION": g.positions(b1v), "TEXCOORD_0": g.accessor(b1uv, 5126, "VEC2")},
                "indices": g.indices(b1f)},
               {"attributes": {"POSITION": g.positions(b2v), "TEXCOORD_0": g.accessor(b2uv, 5126, "VEC2")},
                "indices": g.indices(b2f), "material": 2}]
    nodes = [_node((0.5, 0, 0), Rotation.from_euler("z", 30, degrees=True).as_quat(), (1, 1, 1)),
             _node((0, 1, 0), (0, 0, 0, 1), (-1, 1, 1)),
             _node((0, 0, 2), Rotation.from_euler("x", 90, degrees=True).as_quat(), (2, 2, 2))]
    nodes[0]["mesh"], nodes[1]["mesh"], nodes[2]["mesh"] = 0, 1, 0
    materials = [{"name": "skin", "pbrMetallicRoughness": {"baseColorTexture": {"index": 0}}},
                 {"name": "cloth", "pbrMetallicRoughness": {"baseColorTexture": {"index": 1}, "baseColorFactor": [1, 0.5, 0.5, 1]}},
                 {"name": "paint", "pbrMetallicRoughness": {"baseColorFactor": [0.1, 0.9, 0.2, 1]}}]
    path = g.save(tmp_path / "multi.glb", scene=0, scenes=[{"nodes": [0, 1, 2]}], nodes=nodes,
                  meshes=[{"primitives": prims_a}, {"primitives": prims_b}], materials=materials,
                  textures=[{"sampler": 0, "source": 0}, {"sampler": 0, "source": 0, "name": "again"}],
                  samplers=[{"magFilter": 9728, "wrapS": 33071}], images=[{"bufferView": image_view, "mimeType": "image/png"}])
    strip_f = np.array([[0, 1, 2], [1, 3, 2], [2, 3, 4]])   # glTF 2.0 §3.7.2.1
    parts = [(a0v, a0uv, a0f, nodes[0], 0), (a1v, None, strip_f, nodes[0], 1), (b1v, b1uv, b1f, nodes[1], None),
             (b2v, b2uv, b2f, nodes[1], 2), (a0v, a0uv, a0f, nodes[2], 0), (a1v, None, strip_f, nodes[2], 1)]
    verts, faces, uv, n = [], [], [], 0
    for v, t, f, node, _ in parts:
        w = _world(node)
        verts.append(v.astype(np.float64) @ w[:3, :3].T + w[:3, 3])
        faces.append((f[:, ::-1] if np.linalg.det(w[:3, :3]) < 0 else f) + n)
        uv.append(np.zeros((len(v), 2), f32) if t is None else t)
        n += len(v)
    counts_v, counts_f = [len(p[0]) for p in parts], [len(p[2]) for p in parts]
    want = dict(vertices=np.concatenate(verts), faces=np.concatenate(faces), uv=np.concatenate(uv),
                vertex_ranges=np.stack([np.cumsum(counts_v) - counts_v, counts_v], 1),
                face_ranges=np.stack([np.cumsum(counts_f) - counts_f, counts_f], 1),
                has_uv=np.array([p[1] is not None for p in parts]), primitive_material=[p[4] for p in parts],
                materials=materials, image=img)
    return path, want


def test_hand_built_file_reads_every_primitive_and_material(built):
    path, want = built
    mesh = load_glb(path)
    vis = mesh.visual
    assert isinstance(vis, GltfMultiVisual)
    np.testing.assert_allclose(mesh.vertices, want["vertices"], rtol=0, atol=1e-12)
    assert np.array_equal(mesh.faces, want["faces"])
    for key in ("vertex_ranges", "face_ranges", "uv", "has_uv"):
        got = getattr(vis, key)
        assert np.array_equal(got, want[key]) and got.dtype == np.asarray(want[key]).dtype, key
    assert vis.vertex_ranges.dtype == vis.face_ranges.dtype == np.int64 and vis.uv.dtype == np.float32
    assert vis.primitive_material == want["primitive_material"] and vis.materials == want["materials"]
    assert vis.textures == [{"sampler": 0, "source": 0}, {"sampler": 0, "source": 0, "name": "again"}]
    assert vis.samplers == [{"magFilter": 9728, "wrapS": 33071}]                     # one sampler, one image, stored once
    assert vis.images == [{"mimeType": "image/png"}] and vis.image_bytes == [want["image"]]


def test_the_multi_primitive_warning_is_gone(built, caplog):
    with caplog.at_level(logging.WARNING, logger="actionmesh_b200.gltf"):
        load_glb(built[0])
    assert not [r for r in caplog.records if r.levelno >= logging.WARNING]


def test_files_without_uvs_or_materials_and_single_primitives_are_unchanged(tmp_path):
    rng = np.random.default_rng(3)
    g = Glb()
    prims = [{"attributes": {"POSITION": g.positions(rng.standard_normal((4, 3)))}, "indices": g.indices([0, 1, 2, 1, 2, 3])}
             for _ in range(2)]
    path = g.save(tmp_path / "plain.glb", meshes=[{"primitives": prims}], nodes=[{"mesh": 0}])
    assert load_glb(path).visual is None
    one = Mesh(vertices=rng.standard_normal((5, 3)), faces=np.array([[0, 1, 2], [2, 3, 4]]),
               visual=GltfVisual(uv=rng.random((5, 2)).astype(f32), material={"name": "m"}))
    write_glb(tmp_path / "one.glb", one)
    assert isinstance(load_glb(tmp_path / "one.glb").visual, GltfVisual)


def _same_visual(a, b):
    for key in ("vertex_ranges", "face_ranges", "uv", "has_uv"):
        assert np.array_equal(getattr(a, key), getattr(b, key)), key
    for key in ("primitive_material", "materials", "textures", "samplers", "images", "image_bytes"):
        assert getattr(a, key) == getattr(b, key), key


def test_write_then_load_round_trips(built, tmp_path):
    mesh = load_glb(built[0])
    write_glb(tmp_path / "back.glb", mesh)
    gltf, _ = glb_check.check_glb(tmp_path / "back.glb")
    prims = gltf["meshes"][0]["primitives"]
    assert len(prims) == 6 and ["material" in p for p in prims] == [True, True, False, True, True, True]
    assert ["TEXCOORD_0" in p["attributes"] for p in prims] == list(mesh.visual.has_uv)
    assert len(gltf["images"]) == 1
    back = load_glb(tmp_path / "back.glb")
    assert np.array_equal(back.vertices, mesh.vertices.astype(f32)) and np.array_equal(back.faces, mesh.faces)
    _same_visual(back.visual, mesh.visual)


def _frames(mesh, T=4):
    rng = np.random.default_rng(11)
    return np.stack([np.asarray(mesh.vertices) + 0.05 * k * rng.standard_normal(mesh.vertices.shape) for k in range(T)])


def _read_prims(path):
    gltf, binary = glb_check.check_glb(path)
    acc = lambda i: glb_check.accessor(gltf, binary, i)  # noqa: E731
    return gltf, acc, gltf["meshes"][0]["primitives"]


def _check_materials_and_ranges(gltf, acc, prims, vis, faces):
    assert len(prims) == len(vis.vertex_ranges)
    for p, prim in enumerate(prims):
        (v0, nv), (f0, nf) = vis.vertex_ranges[p], vis.face_ranges[p]
        assert np.array_equal(acc(prim["indices"]).reshape(-1, 3).astype(np.int64) + v0, faces[f0:f0 + nf])
        assert ("TEXCOORD_0" in prim["attributes"]) == vis.has_uv[p]
        if vis.has_uv[p]:
            assert np.array_equal(acc(prim["attributes"]["TEXCOORD_0"]), vis.uv[v0:v0 + nv])
        m = vis.primitive_material[p]
        assert gltf["materials"][prim["material"]] == (DEFAULT_MATERIAL if m is None else vis.materials[m])


def test_animated_glb_per_primitive(built, tmp_path):
    mesh = load_glb(built[0])
    vis, T = mesh.visual, 4
    v = _frames(mesh, T)
    write_animated_glb(tmp_path / "anim.glb", v, mesh.faces, visual=vis)
    gltf, acc, prims = _read_prims(tmp_path / "anim.glb")
    _check_materials_and_ranges(gltf, acc, prims, vis, mesh.faces)
    assert gltf["meshes"][0]["weights"] == [1.0] + [0.0] * (T - 1)
    assert gltf["meshes"][0]["extras"]["targetNames"] == [f"Frame_{k}" for k in range(T)]
    want = v @ ANIMATED_GLB_MAP.T
    for p, prim in enumerate(prims):
        v0, nv = vis.vertex_ranges[p]
        assert len(prim["targets"]) == T
        base = acc(prim["attributes"]["POSITION"]).astype(np.float64)
        for k in range(T):
            got = base + acc(prim["targets"][k]["POSITION"]).astype(np.float64)
            assert np.abs(got - want[k, v0:v0 + nv]).max() <= 2.0 ** -22 * np.abs(want).max()
    morph = sum(gltf["bufferViews"][gltf["accessors"][t["POSITION"]]["bufferView"]]["byteLength"]
                for prim in prims for t in prim["targets"])
    assert morph == 12 * T * len(mesh.vertices)


def test_skinned_glb_per_primitive(built, tmp_path):
    mesh = load_glb(built[0])
    vis = mesh.visual
    v = _frames(mesh, 3)
    fit = as_fit(v, sref.fit(v, 3, 1))
    write_skinned_glb(tmp_path / "skin.glb", fit, mesh.faces, visual=vis)
    gltf, acc, prims = _read_prims(tmp_path / "skin.glb")
    _check_materials_and_ranges(gltf, acc, prims, vis, mesh.faces)
    w = fit.weights / fit.weights.sum(1, keepdims=True)
    for p, prim in enumerate(prims):
        rows = slice(vis.vertex_ranges[p][0], vis.vertex_ranges[p].sum())
        assert np.array_equal(acc(prim["attributes"]["JOINTS_0"]), fit.joints[rows].astype(np.uint8))
        assert np.array_equal(acc(prim["attributes"]["WEIGHTS_0"]), w[rows].astype(f32))
        assert np.array_equal(acc(prim["attributes"]["POSITION"]), (fit.rest[rows] @ ANIMATED_GLB_MAP.T).astype(f32))
    assert gltf["nodes"][0]["skin"] == 0 and len(gltf["skins"]) == 1


@pytest.mark.parametrize("breakage", ["vertex_count", "face_gap", "face_outside", "material", "fields"])
def test_mismatched_ranges_raise_before_writing(built, tmp_path, breakage):
    import copy

    mesh = load_glb(built[0])
    vis = copy.deepcopy(mesh.visual)
    if breakage == "vertex_count":
        vis.vertex_ranges[-1, 1] += 1
    elif breakage == "face_gap":
        vis.face_ranges[1, 0] += 1
    elif breakage == "face_outside":
        mesh.faces[0, 0] = vis.vertex_ranges[1, 0]                   # primitive 0's face reaches primitive 1's vertices
    elif breakage == "material":
        vis.primitive_material[0] = 7
    else:
        vis.has_uv = vis.has_uv[:-1]
    v = _frames(mesh, 2)
    writers = {"a.glb": lambda p: write_glb(p, Mesh(mesh.vertices, mesh.faces, vis)),
               "b.glb": lambda p: write_animated_glb(p, v, mesh.faces, visual=vis),
               "c.glb": lambda p: write_skinned_glb(p, as_fit(v, sref.fit(v, 2, 1)), mesh.faces, visual=vis)}
    for name, write in writers.items():
        with pytest.raises(ValueError, match="visual"):
            write(tmp_path / name)
        assert not (tmp_path / name).exists()


# ---- shading records -------------------------------------------------------------------------------------------------------
def _record_visual():
    rng = np.random.default_rng(2)
    images = [png(rng.integers(0, 255, (3, 5, 3), dtype=np.uint8)), png(rng.integers(0, 255, (2, 2, 3), dtype=np.uint8))]
    materials = [{"pbrMetallicRoughness": {"baseColorTexture": {"index": 0}}},
                 {"pbrMetallicRoughness": {"baseColorTexture": {"index": 0, "texCoord": 1}, "baseColorFactor": [0.5, 0.5, 0.5, 1]}},
                 {"pbrMetallicRoughness": {"baseColorFactor": [0.1, 0.2, 0.3, 1]}},
                 {"pbrMetallicRoughness": {"baseColorTexture": {"index": 1}}},
                 {"pbrMetallicRoughness": {"baseColorTexture": {"index": 2}}}]
    prims = [(0, True), (0, True), (0, False), (1, True), (1, True), (None, False), (None, True), (2, True), (3, True),
             (4, True)]
    P = len(prims)
    return GltfMultiVisual(vertex_ranges=np.stack([3 * np.arange(P), np.full(P, 3)], 1),
                           face_ranges=np.stack([np.arange(P), np.ones(P, np.int64)], 1), uv=rng.random((3 * P, 2)).astype(f32),
                           has_uv=np.array([h for _, h in prims]), primitive_material=[m for m, _ in prims], materials=materials,
                           textures=[{"source": 0}, {"source": 0, "sampler": 0}, {"source": 1}],
                           samplers=[{"magFilter": 9728, "minFilter": 9728, "wrapS": 33071, "wrapT": 33648}],
                           images=[{"mimeType": "image/png"}] * 2, image_bytes=images)


def test_one_record_per_material_and_uv_pair(caplog, monkeypatch):
    vis = _record_visual()
    decoded = []
    real = render._decode
    monkeypatch.setattr(render, "_decode", lambda data: decoded.append(data) or real(data))
    with caplog.at_level(logging.WARNING, logger="actionmesh_b200.render"):
        sh = render.texture_shading(vis)
    assert isinstance(sh, render.MaterialShading)
    # (0, uv) (0, no uv) (1, uv) (None, no uv) (None, uv) (2, uv) (3, uv) (4, uv)
    assert np.array_equal(sh.face_record, [0, 0, 1, 2, 2, 3, 4, 5, 6, 7]) and sh.face_record.dtype == np.int32
    assert len(sh.records) == 8 and len(sh.images) == 2 and decoded == vis.image_bytes
    blue = tuple(DEFAULT_MATERIAL["pbrMetallicRoughness"]["baseColorFactor"][:3])
    r = sh.records
    assert r[0].image == 0 and r[0].base_color == (1.0, 1.0, 1.0)
    assert r[1].image is None and r[2].image is None and r[2].base_color == (0.5, 0.5, 0.5)      # no UVs; texCoord 1
    assert r[3].image is None and r[4].image is None and r[3].base_color == r[4].base_color == blue
    assert r[5].image is None and r[5].base_color == (0.1, 0.2, 0.3)
    assert r[6].image == 0 and (r[6].mag_filter, r[6].min_filter, r[6].wrap_s, r[6].wrap_t) == (9728, 9728, 33071, 33648)
    assert r[7].image == 1 and (r[7].mag_filter, r[7].min_filter, r[7].wrap_s, r[7].wrap_t) == (9729, 9985, 10497, 10497)
    warnings = [x.getMessage() for x in caplog.records if x.levelno == logging.WARNING]
    assert len(warnings) == 2 and "material 0" in warnings[0] and "no UVs" in warnings[0]
    assert "material 1" in warnings[1] and "texCoord 1" in warnings[1]                  # once, for two primitives


def test_one_chain_per_distinct_image(monkeypatch):
    """The level buffer holds each distinct image's chain once, back to back, and every record points into it."""
    vis = _record_visual()
    chains, packed = [], []

    def texture_levels(image, out=None, offset=0):
        chains.append((tuple(image.shape), offset))
        return out, [(offset + o, w, h) for o, w, h in ops.texture_level_table(image.shape[1], image.shape[0])]

    monkeypatch.setattr(ops, "texture_levels", texture_levels)
    monkeypatch.setattr(ops, "shade_records", lambda rows, levels, device: packed.append((rows, levels)) or "records")
    vis_r = render.B200MeshVisualizer(device="cpu")
    sh = render.texture_shading(vis)
    tables = vis_r._material_tables(sh, vis.uv)
    first = ops.texture_chain_bytes(5, 3)
    assert chains == [((3, 5, 3), 0), ((2, 2, 3), first)]
    (rows, levels), = packed
    assert levels.numel() == first + ops.texture_chain_bytes(2, 2) and tables["levels"] is levels
    assert rows[0][0][0] == (0, 5, 3) and rows[6][0] == rows[0][0] and rows[7][0][0] == (first, 2, 2)
    assert all(row[0] is None for row in rows[1:6])
    assert np.array_equal(tables["uv"].numpy(), vis.uv)


def test_record_packing_matches_the_header(tmp_path, amb_lib):
    """ops' record dtype has the C compiler's offsets and size of struct amb_shade_record."""
    import os
    import subprocess

    from conftest import ROOT

    names = ops.SHADE_RECORD.names
    src = tmp_path / "rec.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "actionmesh_b200.h"\nint main(void) {\n'
                   'printf("%zu\\n", sizeof(struct amb_shade_record));\n'
                   + "".join(f'printf("%zu\\n", offsetof(struct amb_shade_record, {n}));\n' for n in names) + "return 0;\n}\n")
    subprocess.run(["cc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(tmp_path / "rec")], check=True)
    got = [int(x) for x in subprocess.run([str(tmp_path / "rec")], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [ops.SHADE_RECORD.itemsize] + [ops.SHADE_RECORD.fields[n][1] for n in names]


def test_records_and_face_records_are_checked_on_the_host():
    from actionmesh_b200 import AmbError

    table = ops.texture_level_table(4, 2)
    size = ops.texture_chain_bytes(4, 2)
    levels = torch.zeros(size, dtype=torch.uint8)
    good = (table, 9729, 9985, 10497, 10497, (1, 1, 1))
    packed = ops.shade_records([good, (None, 9728, 9728, 33071, 33648, (0.5, 0.25, 1))], levels, "cpu")
    assert packed.shape == (2, 272) and packed.dtype == torch.uint8
    rec = packed.numpy().view(ops.SHADE_RECORD)[:, 0]
    assert rec[0]["n_levels"] == len(table) and rec[1]["n_levels"] == 0 and tuple(rec[1]["base_color"]) == (0.5, 0.25, 1)
    assert [tuple(x) for x in zip(rec[0]["level_offset"], rec[0]["level_width"], rec[0]["level_height"])][:len(table)] == table
    for bad in ([], [good] * 65537, [(table, 9730, 9985, 10497, 10497, (1, 1, 1))],
                [(table[:-1], 9729, 9985, 10497, 10497, (1, 1, 1))],
                [([(o + 1, w, h) for o, w, h in table], 9729, 9985, 10497, 10497, (1, 1, 1))]):
        with pytest.raises(AmbError, match="shade_records"):
            ops.shade_records(bad, levels, "cpu")
    assert ops.face_records(np.array([0, 1, 1]), 2, "cpu").dtype == torch.int32
    for bad in (np.array([0, 2]), np.array([-1]), np.array([0.5])):
        with pytest.raises(AmbError, match="face_records"):
            ops.face_records(bad, 2, "cpu")


def test_render_refuses_ranges_that_do_not_fit():
    vis = _record_visual()
    mesh = Mesh(vertices=np.random.default_rng(0).standard_normal((30, 3)), faces=np.arange(30).reshape(10, 3))
    with pytest.raises(ValueError, match="render: visual"):
        render.B200MeshVisualizer(device="cpu").render_frames([Mesh(mesh.vertices[:29], mesh.faces[:9])],
                                                              modalities=("texture",), visual=vis)


def test_material_entry_point_argument_validation(amb_lib):
    """amb_render_shade_materials checks pointers, strides and the record count before any launch (fake pointers)."""
    P = 16
    err = lambda: amb_lib.amb_last_error().decode()  # noqa: E731
    sh = lambda **k: amb_lib.amb_render_shade_materials(  # noqa: E731
        P, 3, P, 1, P, P, P, 3, 2.0, 8, P, k.get("fr", P), k.get("rec", P), k.get("n", 3), P, k.get("out", P),
        k.get("row", 72), k.get("view", 24), None)
    for bad in ("fr", "rec", "out"):
        assert sh(**{bad: None}) < 0 and "null pointer" in err()
    assert sh(row=23) < 0 and "bad strides" in err()
    assert sh(n=0) < 0 and "n_records" in err()
    assert sh(n=65537) < 0 and "n_records" in err()


# ---- the command line ------------------------------------------------------------------------------------------------------
def test_cli_hands_the_multi_visual_to_both_writers_and_the_renderer(built, stubs, frames_dir, tmp_path, monkeypatch,
                                                                     caplog):
    from actionmesh_b200 import inference, skinning

    monkeypatch.setattr(skinning, "fit_skinning", lambda v, n, device=None: as_fit(v, sref.fit(v, n, 1)))
    with caplog.at_level(logging.WARNING):
        inference.main(["--input", str(frames_dir), "--mesh_input", built[0], "--output_dir", str(tmp_path / "out"),
                        "--render_texture", "--skinning_bones", "4"])
    assert not [r for r in caplog.records if "not merged" in r.getMessage()]
    want = load_glb(built[0])
    (r,) = rendered = stubs[1]
    assert rendered and r["modalities"] == ("normal", "texture")
    _same_visual(r["visual"], want.visual)
    for name in ("animated_mesh.glb", "skinned_mesh.glb"):
        gltf, acc, prims = _read_prims(tmp_path / "out" / name)
        _check_materials_and_ranges(gltf, acc, prims, want.visual, want.faces)
        assert glb_check.image_bytes(gltf, glb_check.check_glb(tmp_path / "out" / name)[1]) == want.visual.image_bytes


from test_render_texture_cpu import frames_dir, stubs  # noqa: E402,F401  (the command line's stubbed pipelines)
