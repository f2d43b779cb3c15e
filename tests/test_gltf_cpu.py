"""GLB reading and writing (`actionmesh_b200.gltf`) and `save_deformation`, against numpy restatements.  Every file the
writers produce passes `glb_check.check_glb`, the structural rules of glTF 2.0."""
import base64
import json
import os
import struct

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import glb_check
from actionmesh_b200.gltf import GltfVisual, load_glb, save_deformation, save_meshes, write_animated_glb, write_glb
from actionmesh_b200.pipeline import Mesh
from conftest import GOLDEN

# The layout of a file written by Blender's glTF exporter (Khronos glTF Blender I/O 4.4), with a subset of the reference's
# panda example as its data (tools/gen_gltf_golden.py): u16 indices, NORMAL, a JPEG texture, one bufferView per attribute.
PANDA = os.path.join(GOLDEN, "panda_blender_small.glb")


def _random_mesh(n_faces, n_verts, seed):
    rng = np.random.default_rng(seed)
    return Mesh(vertices=rng.standard_normal((n_verts, 3)) * 0.3, faces=rng.integers(0, n_verts, (n_faces, 3)))


class Glb:
    """A hand-built GLB: arrays appended to one BIN buffer, the JSON written by the test."""

    def __init__(self):
        self.bin, self.gltf = bytearray(), {"asset": {"version": "2.0"}, "bufferViews": [], "accessors": []}

    def view(self, data: bytes, stride=None) -> int:
        self.bin += b"\0" * (-len(self.bin) % 4)
        v = {"buffer": 0, "byteOffset": len(self.bin), "byteLength": len(data)}
        if stride:
            v["byteStride"] = stride
        self.bin += data
        self.gltf["bufferViews"].append(v)
        return len(self.gltf["bufferViews"]) - 1

    def accessor(self, arr, component, type_, view=None, offset=0, count=None, normalized=False) -> int:
        arr = np.asarray(arr)
        if view is None:
            view = self.view(np.ascontiguousarray(arr, glb_check.DTYPES[component]).tobytes())
        acc = {"bufferView": view, "byteOffset": offset, "componentType": component, "type": type_,
               "count": int(count if count is not None else arr.shape[0])}
        if normalized:
            acc["normalized"] = True
        self.gltf["accessors"].append(acc)
        return len(self.gltf["accessors"]) - 1

    def positions(self, v) -> int:
        return self.accessor(np.asarray(v, np.float32), 5126, "VEC3")

    def indices(self, f, component=5125) -> int:
        return self.accessor(np.asarray(f).reshape(-1), component, "SCALAR")

    def save(self, path, **extra) -> str:
        gltf = {**self.gltf, **extra}
        self.bin += b"\0" * (-len(self.bin) % 4)
        if "buffers" not in gltf:
            gltf["buffers"] = [{"byteLength": len(self.bin)}]
        js = json.dumps(gltf).encode()
        js += b" " * (-len(js) % 4)
        body = struct.pack("<II", len(js), 0x4E4F534A) + js
        if self.bin and "uri" not in gltf["buffers"][0]:
            body += struct.pack("<II", len(self.bin), 0x004E4942) + bytes(self.bin)
        with open(path, "wb") as fh:
            fh.write(b"glTF" + struct.pack("<II", 2, 12 + len(body)) + body)
        return str(path)


def _trs(t=(0, 0, 0), q=(0, 0, 0, 1), s=(1, 1, 1)):
    m = np.eye(4)
    m[:3, :3] = Rotation.from_quat(q).as_matrix() @ np.diag(s)
    m[:3, 3] = t
    return m


def _apply(m, v):
    return (np.c_[np.asarray(v, np.float32).astype(np.float64), np.ones(len(v))] @ m.T)[:, :3]


def _tri(seed, n_verts=7, n_faces=5):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((n_verts, 3)).astype(np.float32), rng.integers(0, n_verts, (n_faces, 3))


# ---------------------------------------------------------------------------------------------------------- round trips
@pytest.mark.parametrize("n_faces,n_verts", [(1, 3), (1000, 520), (70000, 70000)])
def test_write_then_load_round_trips(tmp_path, n_faces, n_verts):
    mesh = _random_mesh(n_faces, n_verts, seed=n_faces)
    path = tmp_path / "m.glb"
    write_glb(path, mesh)
    gltf, _ = glb_check.check_glb(path)
    assert len(gltf["meshes"]) == len(gltf["nodes"]) == len(gltf["scenes"]) == 1
    assert gltf["accessors"][gltf["meshes"][0]["primitives"][0]["indices"]]["componentType"] == 5125
    back = load_glb(path)
    assert back.vertices.dtype == np.float64 and back.faces.dtype == np.int64
    assert np.array_equal(back.vertices, mesh.vertices.astype(np.float32)) and np.array_equal(back.faces, mesh.faces)
    assert back.visual is None


def test_zero_faces_writes_a_valid_file_that_has_no_geometry(tmp_path):
    path = tmp_path / "empty.glb"
    write_glb(path, Mesh(vertices=np.zeros((4, 3)), faces=np.zeros((0, 3), np.int64)))
    gltf, binary = glb_check.check_glb(path)
    assert gltf["scenes"] == [{"nodes": [0]}] and gltf["nodes"] == [{}] and binary == b""
    with pytest.raises(ValueError, match="No mesh geometry found"):
        load_glb(path)


def test_save_meshes_names_files_and_accepts_any_mesh_object(tmp_path):
    class Duck:                                          # anything with .vertices / .faces, as trimesh objects have
        def __init__(self, m):
            self.vertices, self.faces = m.vertices, m.faces

    meshes = [_random_mesh(20, 12, seed=s) for s in range(3)]
    paths = save_meshes([meshes[0], Duck(meshes[1]), meshes[2]], tmp_path / "out")
    assert sorted(os.listdir(tmp_path / "out")) == ["mesh_00.glb", "mesh_01.glb", "mesh_02.glb"]
    for p, m in zip(paths, meshes):
        glb_check.check_glb(p)
        assert np.array_equal(load_glb(p).vertices, m.vertices.astype(np.float32))


# ---------------------------------------------------------------------------------------------------- hand-built files
def test_node_hierarchy_mixing_matrix_and_trs(tmp_path):
    (va, fa), (vb, fb) = _tri(1), _tri(2)
    g = Glb()
    ma = {"primitives": [{"attributes": {"POSITION": g.positions(va)}, "indices": g.indices(fa)}]}
    mb = {"primitives": [{"attributes": {"POSITION": g.positions(vb)}, "indices": g.indices(fb)}]}
    q0, q2 = Rotation.from_euler("xyz", [0.3, -0.7, 1.1]).as_quat(), Rotation.from_euler("zyx", [2.0, 0.1, -0.4]).as_quat()
    m1 = _trs((0.5, -1, 2), Rotation.from_euler("y", 0.9).as_quat(), (1.5, 1.5, 0.5))
    nodes = [{"translation": [1, 2, 3], "rotation": q0.tolist(), "scale": [2, 1, 0.5], "mesh": 0, "children": [1]},
             {"matrix": m1.T.reshape(-1).tolist(), "children": [2]},
             {"translation": [-1, 0, 0.25], "rotation": q2.tolist(), "mesh": 1},
             {"mesh": 1, "scale": [-1, 1, 1]}]            # mirrored: its triangles are reversed
    path = g.save(tmp_path / "h.glb", meshes=[ma, mb], nodes=nodes, scenes=[{"nodes": [0, 3]}], scene=0)
    w0 = _trs((1, 2, 3), q0, (2, 1, 0.5))
    w2 = w0 @ m1 @ _trs((-1, 0, 0.25), q2)
    w3 = _trs(s=(-1, 1, 1))
    got = load_glb(path)
    want_v = np.concatenate([_apply(w0, va), _apply(w2, vb), _apply(w3, vb)])
    want_f = np.concatenate([fa, fb + 7, fb[:, ::-1] + 14])
    np.testing.assert_allclose(got.vertices, want_v, rtol=0, atol=1e-12)
    assert np.array_equal(got.faces, want_f)


def test_default_scene_fallbacks(tmp_path):
    (va, fa), (vb, fb) = _tri(3), _tri(4)
    g = Glb()
    meshes = [{"primitives": [{"attributes": {"POSITION": g.positions(v)}, "indices": g.indices(f)}]}
              for v, f in ((va, fa), (vb, fb))]
    nodes = [{"mesh": 0, "children": [1]}, {"mesh": 1, "translation": [0, 0, 1]}, {"mesh": 1}]
    # no `scene`: scene 0 (node 2 only)
    one = load_glb(g.save(tmp_path / "a.glb", meshes=meshes, nodes=nodes, scenes=[{"nodes": [2]}, {"nodes": [0]}]))
    assert np.array_equal(one.vertices, vb.astype(np.float64)) and np.array_equal(one.faces, fb)
    # no scenes: every root node (0 with its child 1, then 2)
    roots = load_glb(g.save(tmp_path / "b.glb", meshes=meshes, nodes=nodes))
    va64, vb64 = va.astype(np.float64), vb.astype(np.float64)
    assert np.array_equal(roots.vertices, np.concatenate([va64, vb64 + [0, 0, 1], vb64]))
    assert np.array_equal(roots.faces, np.concatenate([fa, fb + 7, fb + 14]))


def test_mesh_instanced_by_two_nodes_appears_twice(tmp_path):
    v, f = _tri(5)
    g = Glb()
    mesh = {"primitives": [{"attributes": {"POSITION": g.positions(v)}, "indices": g.indices(f)}]}
    path = g.save(tmp_path / "i.glb", meshes=[mesh], nodes=[{"mesh": 0}, {"mesh": 0, "translation": [3, 0, 0]}],
                  scenes=[{"nodes": [0, 1]}], scene=0)
    got = load_glb(path)
    v64 = v.astype(np.float64)
    assert np.array_equal(got.vertices, np.concatenate([v64, v64 + [3, 0, 0]]))
    assert np.array_equal(got.faces, np.concatenate([f, f + len(v)]))


def test_interleaved_position_and_uv(tmp_path):
    v, f = _tri(6)
    uv = np.random.default_rng(6).random((len(v), 2)).astype(np.float32)
    g = Glb()
    inter = np.concatenate([v, uv], axis=1).astype(np.float32)        # 20-byte vertices: xyz uv
    view = g.view(inter.tobytes(), stride=20)
    pos = g.accessor(v, 5126, "VEC3", view=view, offset=0)
    tex = g.accessor(uv, 5126, "VEC2", view=view, offset=12)
    mesh = {"primitives": [{"attributes": {"POSITION": pos, "TEXCOORD_0": tex}, "indices": g.indices(f)}]}
    got = load_glb(g.save(tmp_path / "s.glb", meshes=[mesh], nodes=[{"mesh": 0}], scenes=[{"nodes": [0]}]))
    assert np.array_equal(got.vertices, v.astype(np.float64)) and np.array_equal(got.faces, f)
    assert got.visual.uv.dtype == np.float32 and np.array_equal(got.visual.uv, uv) and got.visual.material is None


@pytest.mark.parametrize("component", [5121, 5123, 5125])
def test_index_widths_and_normalized_uvs(tmp_path, component):
    v, f = _tri(7, n_verts=9, n_faces=11)
    rng = np.random.default_rng(7)
    g = Glb()
    uv_dtype = {5121: np.uint8, 5123: np.uint16, 5125: np.float32}[component]
    uv = (rng.random((len(v), 2)) * (np.iinfo(uv_dtype).max if uv_dtype != np.float32 else 1)).astype(uv_dtype)
    tex = g.accessor(uv, {np.uint8: 5121, np.uint16: 5123, np.float32: 5126}[uv_dtype], "VEC2",
                     normalized=uv_dtype != np.float32)
    mesh = {"primitives": [{"attributes": {"POSITION": g.positions(v), "TEXCOORD_0": tex},
                            "indices": g.indices(f, component)}]}
    got = load_glb(g.save(tmp_path / "u.glb", meshes=[mesh], nodes=[{"mesh": 0}], scenes=[{"nodes": [0]}]))
    assert np.array_equal(got.faces, f)
    scale = 1.0 if uv_dtype == np.float32 else float(np.iinfo(uv_dtype).max)
    assert np.array_equal(got.visual.uv, (uv.astype(np.float64) / scale).astype(np.float32))


def test_non_indexed_strip_fan_and_points(tmp_path):
    rng = np.random.default_rng(8)
    v = [rng.standard_normal((n, 3)).astype(np.float32) for n in (6, 7, 6, 5)]
    g = Glb()
    prims = [{"attributes": {"POSITION": g.positions(v[0])}},                                   # non-indexed list
             {"attributes": {"POSITION": g.positions(v[1])}, "indices": g.indices(np.arange(7)[::-1], 5123), "mode": 5},
             {"attributes": {"POSITION": g.positions(v[2])}, "mode": 6},
             {"attributes": {"POSITION": g.positions(v[3])}, "mode": 0}]                          # points: skipped
    got = load_glb(g.save(tmp_path / "p.glb", meshes=[{"primitives": prims}], nodes=[{"mesh": 0}],
                          scenes=[{"nodes": [0]}]))
    strip_idx = np.arange(7)[::-1]
    strip = [(strip_idx[i], strip_idx[i + 1 + i % 2], strip_idx[i + 2 - i % 2]) for i in range(5)]
    fan = [(i + 1, i + 2, 0) for i in range(4)]
    want_f = np.concatenate([np.arange(6).reshape(2, 3), np.array(strip) + 6, np.array(fan) + 13])
    assert np.array_equal(got.vertices, np.concatenate(v[:3]).astype(np.float64))
    assert np.array_equal(got.faces, want_f)
    only_points = Glb()
    mesh = {"primitives": [{"attributes": {"POSITION": only_points.positions(v[3])}, "mode": 0}]}
    with pytest.raises(ValueError, match="No mesh geometry found"):
        load_glb(only_points.save(tmp_path / "pts.glb", meshes=[mesh], nodes=[{"mesh": 0}], scenes=[{"nodes": [0]}]))


def test_data_uri_buffer(tmp_path):
    v, f = _tri(9)
    g = Glb()
    mesh = {"primitives": [{"attributes": {"POSITION": g.positions(v)}, "indices": g.indices(f)}]}
    payload = bytes(g.bin) + b"\0" * (-len(g.bin) % 4)
    uri = "data:application/octet-stream;base64," + base64.b64encode(payload).decode()
    path = g.save(tmp_path / "d.glb", meshes=[mesh], nodes=[{"mesh": 0}], scenes=[{"nodes": [0]}],
                  buffers=[{"byteLength": len(payload), "uri": uri}])
    got = load_glb(path)
    assert np.array_equal(got.vertices, v.astype(np.float64)) and np.array_equal(got.faces, f)


def test_unsupported_files_raise(tmp_path):
    v, f = _tri(10)
    g = Glb()
    mesh = {"primitives": [{"attributes": {"POSITION": g.positions(v)}, "indices": g.indices(f)}]}
    scene = dict(meshes=[mesh], nodes=[{"mesh": 0}], scenes=[{"nodes": [0]}])
    draco = g.save(tmp_path / "draco.glb", extensionsRequired=["KHR_draco_mesh_compression"],
                   extensionsUsed=["KHR_draco_mesh_compression"], **scene)
    with pytest.raises(ValueError, match="KHR_draco_mesh_compression"):
        load_glb(draco)
    good = g.save(tmp_path / "good.glb", **scene)
    data = bytearray(open(good, "rb").read())
    data[:4] = b"glTX"
    (tmp_path / "magic.glb").write_bytes(bytes(data))
    with pytest.raises(ValueError, match="magic"):
        load_glb(tmp_path / "magic.glb")
    data[:4] = b"glTF"
    struct.pack_into("<I", data, 16, 0x12345678)             # first chunk type is not JSON
    (tmp_path / "chunk.glb").write_bytes(bytes(data))
    with pytest.raises(ValueError, match="JSON"):
        load_glb(tmp_path / "chunk.glb")
    g.gltf["accessors"][0]["sparse"] = {"count": 1, "indices": {}, "values": {}}
    with pytest.raises(ValueError, match="sparse"):
        load_glb(g.save(tmp_path / "sparse.glb", **scene))


# ------------------------------------------------------------------------------------------------ a real exporter's file
def test_panda_from_blender(tmp_path):
    gltf, binary = glb_check.check_glb(PANDA)
    assert gltf["asset"]["generator"].startswith("Khronos glTF Blender I/O")
    prim = gltf["meshes"][0]["primitives"][0]
    attrs = prim["attributes"]
    mesh = load_glb(PANDA)
    assert mesh.vertices.shape == (1088, 3) and mesh.faces.shape == (973, 3)
    assert np.array_equal(mesh.vertices, glb_check.accessor(gltf, binary, attrs["POSITION"]).astype(np.float64))
    assert np.array_equal(mesh.faces, glb_check.accessor(gltf, binary, prim["indices"]).reshape(-1, 3).astype(np.int64))
    acc = gltf["accessors"][attrs["POSITION"]]
    assert mesh.vertices.min(0).tolist() == acc["min"] and mesh.vertices.max(0).tolist() == acc["max"]
    vis = mesh.visual
    assert vis.uv.dtype == np.float32 and np.array_equal(vis.uv, glb_check.accessor(gltf, binary, attrs["TEXCOORD_0"]))
    assert vis.images == [{"mimeType": "image/jpeg", "name": "texture"}] and vis.image_bytes[0][:3] == b"\xff\xd8\xff"
    assert vis.image_bytes == glb_check.image_bytes(gltf, binary)
    assert vis.material == gltf["materials"][0] and vis.textures == [{"sampler": 0, "source": 0}]
    assert vis.samplers == gltf["samplers"]
    out = tmp_path / "panda_out.glb"
    write_glb(out, mesh)
    glb_check.check_glb(out)
    back = load_glb(out)
    assert np.array_equal(back.vertices, mesh.vertices) and np.array_equal(back.faces, mesh.faces)
    assert np.array_equal(back.visual.uv, vis.uv) and back.visual.material == vis.material
    assert back.visual.image_bytes == vis.image_bytes and back.visual.textures == vis.textures
    assert back.visual.samplers == vis.samplers


# ---------------------------------------------------------------------------------------------------------- animated GLB
@pytest.mark.parametrize("n_frames,fps", [(1, 8), (16, 8), (31, 24)])
def test_animated_glb_shows_each_frame(tmp_path, n_frames, fps):
    mesh = _random_mesh(300, 200, seed=n_frames)
    rng = np.random.default_rng(n_frames)
    verts = mesh.vertices[None] + 0.05 * np.cumsum(rng.standard_normal((n_frames, 200, 3)), axis=0)
    path = tmp_path / "anim.glb"
    write_animated_glb(path, verts.astype(np.float32), mesh.faces, fps=fps)
    a = glb_check.check_animated(path, verts.astype(np.float32), mesh.faces, fps=fps)
    assert a["material"]["doubleSided"] is True and a["uv"] is None and a["image_bytes"] == []
    pbr = a["material"]["pbrMetallicRoughness"]
    assert pbr == {"baseColorFactor": [0.2, 0.4, 0.8, 1.0], "metallicFactor": 0.1, "roughnessFactor": 0.4}
    assert "NORMAL" not in a["gltf"]["meshes"][0]["primitives"][0]["attributes"]
    assert "extensionsUsed" not in a["gltf"]


def test_animated_glb_keeps_the_texture(tmp_path):
    mesh = load_glb(PANDA)
    rng = np.random.default_rng(11)
    verts = mesh.vertices[None] + 0.01 * rng.standard_normal((4, len(mesh.vertices), 3))
    path = tmp_path / "anim_tex.glb"
    write_animated_glb(path, verts, mesh.faces, fps=8, visual=mesh.visual)
    a = glb_check.check_animated(path, verts, mesh.faces)
    assert np.array_equal(a["uv"], mesh.visual.uv) and a["image_bytes"] == mesh.visual.image_bytes
    assert a["material"] == mesh.visual.material


def test_animated_glb_binary_is_uncompressed_float32(tmp_path):
    n_frames, n_verts, n_faces = 10, 250, 400
    mesh = _random_mesh(n_faces, n_verts, seed=12)
    write_animated_glb(tmp_path / "s.glb", np.repeat(mesh.vertices[None], n_frames, 0), mesh.faces)
    _, binary = glb_check.check_glb(tmp_path / "s.glb")
    # base + one 12-byte delta per vertex and frame, u32 indices, keyframe times, the T x T weights
    assert len(binary) == 12 * n_verts * (1 + n_frames) + 12 * n_faces + 4 * n_frames + 4 * n_frames ** 2


# ------------------------------------------------------------------------------------------------------- save_deformation
def test_save_deformation_restates_the_reference(tmp_path):
    mesh = _random_mesh(50, 30, seed=13)
    rng = np.random.default_rng(13)
    meshes = [Mesh(vertices=mesh.vertices + 0.1 * rng.standard_normal(mesh.vertices.shape), faces=mesh.faces)
              for _ in range(5)]
    vp, fp = save_deformation(meshes, tmp_path / "sub" / "deformations")
    assert (vp.name, fp.name) == ("deformations_vertices.npy", "deformations_faces.npy")
    want = np.stack([m.vertices.astype(np.float32) for m in meshes])[:, :, [2, 0, 1]]
    want[:, :, 0] = -want[:, :, 0]
    got_v, got_f = np.load(vp), np.load(fp)
    assert got_v.dtype == np.float32 and np.array_equal(got_v, want)
    assert got_f.dtype == np.int32 and np.array_equal(got_f, mesh.faces.astype(np.int32))


def test_save_deformation_errors(tmp_path):
    a = _random_mesh(10, 8, seed=14)
    with pytest.raises(ValueError, match="^Cannot save deformation from empty mesh list$"):
        save_deformation([], tmp_path / "d")
    with pytest.raises(ValueError, match=r"^Mesh 1 has 7 vertices, expected 8 \(same as first mesh\)$"):
        save_deformation([a, Mesh(vertices=a.vertices[:7], faces=a.faces)], tmp_path / "d")
    with pytest.raises(ValueError, match="^Mesh 1 has different face topology than the first mesh. All meshes must "
                                         "share the same faces for deformation export.$"):
        save_deformation([a, Mesh(vertices=a.vertices, faces=a.faces[::-1])], tmp_path / "d")


def test_visual_with_wrong_uv_count_is_refused(tmp_path):
    mesh = _random_mesh(10, 8, seed=15)
    mesh.visual = GltfVisual(uv=np.zeros((7, 2), np.float32))
    with pytest.raises(ValueError, match="uv"):
        write_glb(tmp_path / "bad.glb", mesh)
