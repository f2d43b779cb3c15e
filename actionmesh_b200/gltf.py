"""GLB (binary glTF 2.0) files and the deformation arrays, with numpy and the standard library only: the reference's
`actionmesh/io/mesh_io.py` (trimesh) and `actionmesh/io/glb_export.py` (Blender) without either dependency.

  load_glb(path) -> Mesh                     every triangle primitive of the default scene, node transforms applied
  write_glb(path, mesh)                      one node, one mesh, one triangle primitive per material (what trimesh exports)
  write_animated_glb(path, vertices, faces)  one morph target per frame and a weights animation (what Blender exports)
  write_skinned_glb(path, fit, faces)        a rest mesh, its bones and skin weights, and a joint animation
  load_rig(path) -> GltfRig                  a rigged file's skeleton and skin, in load_glb's vertex order
  write_rig_animation(src, out, rig, fit)    the source file plus one joint animation (DESIGN.md §21)
  save_meshes(meshes, output_dir)            mesh_00.glb, mesh_01.glb, ...
  save_deformation(meshes, path)             {stem}_vertices.npy / {stem}_faces.npy

DESIGN.md §19 states the formats, the coordinate map of the animated file and what is not restated.
"""
from __future__ import annotations

import base64
import copy
import json
import logging
import os
import struct
import urllib.parse
from dataclasses import dataclass, field
from pathlib import Path
from typing import Optional

import numpy as np

from .pipeline import Mesh

logger = logging.getLogger(__name__)

GLB_MAGIC = b"glTF"
CHUNK_JSON = 0x4E4F534A
CHUNK_BIN = 0x004E4942
ARRAY_BUFFER, ELEMENT_ARRAY_BUFFER = 34962, 34963
F32, U8, U16, U32 = 5126, 5121, 5123, 5125
COMPONENT_DTYPES = {5120: np.dtype("<i1"), U8: np.dtype("<u1"), 5122: np.dtype("<i2"), U16: np.dtype("<u2"),
                    U32: np.dtype("<u4"), F32: np.dtype("<f4")}
TYPE_SIZES = {"SCALAR": 1, "VEC2": 2, "VEC3": 3, "VEC4": 4, "MAT4": 16}
TRIANGLES, TRIANGLE_STRIP, TRIANGLE_FAN = 4, 5, 6

# (x, y, z) -> (-z, y, -x): `save_deformation`'s (x, y, z) -> (-z, x, y) followed by Blender's +Y-up export
# (bx, by, bz) -> (bx, bz, -by).  det = -1 (DESIGN §19).
ANIMATED_GLB_MAP = np.array([[0.0, 0.0, -1.0], [0.0, 1.0, 0.0], [-1.0, 0.0, 0.0]])

DEFAULT_MATERIAL = {"name": "BlueMaterial", "doubleSided": True,
                    "pbrMetallicRoughness": {"baseColorFactor": [0.2, 0.4, 0.8, 1.0], "metallicFactor": 0.1,
                                             "roughnessFactor": 0.4}}


@dataclass
class GltfVisual:
    """The texture side of a one-primitive glTF mesh, as `load_glb` reads it and the writers write it back.

    uv: (V, 2) float32 TEXCOORD_0 (normalized integer UVs converted to float), or None.
    material: the primitive's glTF material JSON, or None; its texture references index `textures`.
    textures / samplers / images: the glTF JSON of what the material references, re-indexed from 0 (an image entry
    carries `mimeType` and `name` only; its bytes are `image_bytes[i]`)."""
    uv: Optional[np.ndarray] = None
    material: Optional[dict] = None
    textures: list = field(default_factory=list)
    samplers: list = field(default_factory=list)
    images: list = field(default_factory=list)
    image_bytes: list = field(default_factory=list)


@dataclass
class GltfMultiVisual:
    """The texture side of a mesh made of P >= 2 glTF primitives, in `load_glb`'s concatenation order; the writers give each
    primitive back its own range and material (DESIGN §19).

    vertex_ranges / face_ranges: (P, 2) int64 (start, count), contiguous and tiling the mesh's vertices and faces; the faces
    of primitive p index only its vertex range.  uv: (V, 2) float32 TEXCOORD_0 over all vertices (0 on the rows of
    primitives without it), or None when no primitive has one; has_uv: (P,) bool.  primitive_material: P entries, each an
    index into `materials` or None.  materials / textures / samplers / images: the glTF JSON, re-indexed from 0 as in
    `GltfVisual`, each entry stored once however many primitives or textures share it; image i's bytes are `image_bytes[i]`."""
    vertex_ranges: np.ndarray
    face_ranges: np.ndarray
    uv: Optional[np.ndarray] = None
    has_uv: np.ndarray = field(default_factory=lambda: np.zeros(0, bool))
    primitive_material: list = field(default_factory=list)
    materials: list = field(default_factory=list)
    textures: list = field(default_factory=list)
    samplers: list = field(default_factory=list)
    images: list = field(default_factory=list)
    image_bytes: list = field(default_factory=list)


def check_multi_visual(visual: GltfMultiVisual, n_vertices: int, faces: np.ndarray) -> None:
    """ValueError unless `visual`'s ranges tile `n_vertices` vertices and the (F, 3) `faces`, each range non-empty, each
    primitive's faces inside its own vertex range, and its per-primitive fields have P entries."""
    vr, fr = np.asarray(visual.vertex_ranges), np.asarray(visual.face_ranges)
    P = len(vr)
    if vr.shape != (P, 2) or fr.shape != (P, 2) or P < 1:
        raise ValueError(f"visual: vertex_ranges {vr.shape} and face_ranges {fr.shape} must both be (P, 2), P >= 1")
    for name, r, total in (("vertex", vr, n_vertices), ("face", fr, len(faces))):
        starts = np.concatenate([[0], np.cumsum(r[:, 1])[:-1]])
        if (r[:, 1] < 1).any() or not np.array_equal(r[:, 0], starts) or int(r[:, 1].sum()) != total:
            raise ValueError(f"visual: the {name} ranges do not tile the mesh's {total} {name}s")
    if len(np.asarray(visual.has_uv)) != P or len(visual.primitive_material) != P:
        raise ValueError(f"visual: has_uv and primitive_material need {P} entries")
    if any(m is not None and not 0 <= m < len(visual.materials) for m in visual.primitive_material):
        raise ValueError(f"visual: a primitive's material is outside the {len(visual.materials)} materials")
    if visual.uv is not None and np.shape(visual.uv) != (n_vertices, 2):
        raise ValueError(f"visual.uv has shape {np.shape(visual.uv)}, expected ({n_vertices}, 2)")
    if np.asarray(visual.has_uv).any() and visual.uv is None:
        raise ValueError("visual: a primitive has UVs but visual.uv is None")
    if len(faces):
        owner = np.repeat(np.arange(P), fr[:, 1])
        lo, hi = vr[owner, 0], vr[owner, 0] + vr[owner, 1]
        if (faces.min(1) < lo).any() or (faces.max(1) >= hi).any():
            raise ValueError("visual: a face indexes a vertex outside its primitive's range")


# ------------------------------------------------------------------------------------------------------------------ reading
def _parse_glb(data: bytes, path) -> tuple[dict, Optional[bytes]]:
    """(JSON, BIN chunk payload or None) of a GLB file; ValueError on a bad header or chunk layout."""
    if len(data) < 20:
        raise ValueError(f"{path}: too short for a GLB file ({len(data)} bytes)")
    magic, version, length = struct.unpack_from("<4sII", data, 0)
    if magic != GLB_MAGIC:
        raise ValueError(f"{path}: not a GLB file (magic {magic!r}, expected b'glTF')")
    if version != 2:
        raise ValueError(f"{path}: GLB version {version} is not supported (only glTF 2.0)")
    if length > len(data):
        raise ValueError(f"{path}: header length {length} exceeds the file size {len(data)}")
    chunks, off = [], 12
    while off < length:
        if off + 8 > length:
            raise ValueError(f"{path}: truncated chunk header at byte {off}")
        clen, ctype = struct.unpack_from("<II", data, off)
        if off + 8 + clen > length:
            raise ValueError(f"{path}: chunk at byte {off} ({clen} bytes) runs past the end of the file")
        chunks.append((ctype, data[off + 8:off + 8 + clen]))
        off += 8 + clen
    if not chunks or chunks[0][0] != CHUNK_JSON:
        raise ValueError(f"{path}: the first chunk is not JSON")
    try:
        gltf = json.loads(chunks[0][1].decode("utf-8"))
    except (UnicodeDecodeError, json.JSONDecodeError) as exc:
        raise ValueError(f"{path}: the JSON chunk does not parse: {exc}") from exc
    binary = chunks[1][1] if len(chunks) > 1 and chunks[1][0] == CHUNK_BIN else None
    return gltf, binary


class _Reader:
    """Buffers, bufferViews and accessors of one parsed glTF."""

    def __init__(self, gltf: dict, binary: Optional[bytes], path):
        self.gltf, self.binary, self.path = gltf, binary, Path(path)
        self._buffers: dict = {}

    def buffer(self, i: int) -> bytes:
        if i not in self._buffers:
            buf = self.gltf["buffers"][i]
            uri = buf.get("uri")
            if uri is None:
                if i != 0 or self.binary is None:
                    raise ValueError(f"{self.path}: buffer {i} has no uri and no BIN chunk")
                data = self.binary
            else:
                data = _read_uri(uri, self.path)
            if len(data) < buf["byteLength"]:
                raise ValueError(f"{self.path}: buffer {i} holds {len(data)} bytes, byteLength is {buf['byteLength']}")
            self._buffers[i] = data
        return self._buffers[i]

    def view_bytes(self, v: int) -> bytes:
        view = self.gltf["bufferViews"][v]
        start = view.get("byteOffset", 0)
        buf = self.buffer(view["buffer"])
        if start + view["byteLength"] > len(buf):
            raise ValueError(f"{self.path}: bufferView {v} runs past its buffer")
        return buf[start:start + view["byteLength"]]

    def accessor(self, a: int) -> np.ndarray:
        """(count, n) array of accessor `a` in its stored dtype (n = 1 for SCALAR)."""
        acc = self.gltf["accessors"][a]
        if "sparse" in acc:
            raise ValueError(f"{self.path}: accessor {a} is sparse, which is not supported")
        if acc["type"] not in TYPE_SIZES or acc["componentType"] not in COMPONENT_DTYPES:
            raise ValueError(f"{self.path}: accessor {a} has an unsupported type {acc['type']}/{acc['componentType']}")
        dtype, n, count = COMPONENT_DTYPES[acc["componentType"]], TYPE_SIZES[acc["type"]], acc["count"]
        if "bufferView" not in acc:
            return np.zeros((count, n), dtype)           # the spec's all-zero accessor
        view = self.gltf["bufferViews"][acc["bufferView"]]
        data = self.view_bytes(acc["bufferView"])
        elem = n * dtype.itemsize
        stride = view.get("byteStride") or elem
        start = acc.get("byteOffset", 0)
        if count and start + (count - 1) * stride + elem > len(data):
            raise ValueError(f"{self.path}: accessor {a} runs past bufferView {acc['bufferView']}")
        return np.ndarray((count, n), dtype, buffer=data, offset=start, strides=(stride, dtype.itemsize)).copy()

    def float_accessor(self, a: int) -> np.ndarray:
        """Accessor `a` as float, with normalized integer components mapped as the spec defines."""
        acc = self.gltf["accessors"][a]
        x = self.accessor(a)
        if x.dtype.kind == "f" or not acc.get("normalized", False):
            return x.astype(np.float64)
        top = float(np.iinfo(x.dtype).max)
        return np.maximum(x / top, -1.0)


def _read_uri(uri: str, path: Path) -> bytes:
    if uri.startswith("data:"):
        head, _, payload = uri.partition(",")
        if not head.endswith(";base64"):
            return urllib.parse.unquote_to_bytes(payload)
        return base64.b64decode(payload)
    ext = path.parent / urllib.parse.unquote(uri)
    if not ext.is_file():
        raise ValueError(f"{path}: external resource {uri!r} not found next to the file")
    return ext.read_bytes()


def _node_matrix(node: dict) -> np.ndarray:
    """4x4 float64 local transform: `matrix` (column-major) or T * R * S (quaternion x, y, z, w)."""
    if "matrix" in node:
        return np.asarray(node["matrix"], dtype=np.float64).reshape(4, 4).T
    x, y, z, w = np.asarray(node.get("rotation", [0.0, 0.0, 0.0, 1.0]), dtype=np.float64)
    s = x * x + y * y + z * z + w * w
    x, y, z, w = (c / np.sqrt(s) for c in (x, y, z, w)) if s > 0 else (0.0, 0.0, 0.0, 1.0)
    r = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    m = np.eye(4)
    m[:3, :3] = r * np.asarray(node.get("scale", [1.0, 1.0, 1.0]), dtype=np.float64)[None, :]
    m[:3, 3] = node.get("translation", [0.0, 0.0, 0.0])
    return m


def _triangles(idx: np.ndarray, mode: int) -> np.ndarray:
    """(F, 3) triangles of a TRIANGLES / TRIANGLE_STRIP / TRIANGLE_FAN index list (glTF 2.0 §3.7.2.1)."""
    n = len(idx)
    if mode == TRIANGLES:
        return idx[:n - n % 3].reshape(-1, 3)
    if n < 3:
        return np.zeros((0, 3), np.int64)
    k = np.arange(n - 2)
    if mode == TRIANGLE_STRIP:
        return np.stack([idx[k], idx[k + 1 + k % 2], idx[k + 2 - k % 2]], axis=1)
    return np.stack([idx[k + 1], idx[k + 2], np.full_like(k, idx[0])], axis=1)


def _root_nodes(gltf: dict) -> list:
    """The default scene's nodes; scene 0 when `scene` is absent; every root node when there are no scenes."""
    scenes = gltf.get("scenes") or []
    if scenes:
        return list(scenes[gltf.get("scene", 0)].get("nodes", []))
    children = {c for node in gltf.get("nodes", []) for c in node.get("children", [])}
    return [i for i in range(len(gltf.get("nodes", []))) if i not in children]


def _mesh_instances(gltf: dict, path, visited: Optional[dict] = None) -> list:
    """[(mesh index, 4x4 world transform, node index)] in depth-first node order, children in their listed order.  When
    `visited` is a dict it receives node -> (parent node or -1, world transform) for every node reached."""
    nodes, out = gltf.get("nodes", []), []

    def visit(i, parent_i, parent, ancestors):
        if i in ancestors:
            raise ValueError(f"{path}: node {i} is its own ancestor")
        world = parent @ _node_matrix(nodes[i])
        if visited is not None:
            visited[i] = (parent_i, world)
        if "mesh" in nodes[i]:
            out.append((nodes[i]["mesh"], world, i))
        for c in nodes[i].get("children", []):
            visit(c, i, world, ancestors | {i})

    for r in _root_nodes(gltf):
        visit(r, -1, np.eye(4), frozenset())
    return out


class _Collector:
    """Copies materials and what they reference out of one file into `out` (its textures / samplers / images /
    image_bytes lists), re-indexed from 0 in first-use order, each source entry once."""

    def __init__(self, reader: _Reader, out):
        self.reader, self.out = reader, out
        self.tex_map, self.smp_map, self.img_map = {}, {}, {}

    def image(self, i):
        if i not in self.img_map:
            img = self.reader.gltf["images"][i]
            data = (self.reader.view_bytes(img["bufferView"]) if "bufferView" in img
                    else _read_uri(img["uri"], self.reader.path))
            entry = {"mimeType": img.get("mimeType") or _mime_type(data)}
            if "name" in img:
                entry["name"] = img["name"]
            self.img_map[i] = len(self.out.images)
            self.out.images.append(entry)
            self.out.image_bytes.append(bytes(data))
        return self.img_map[i]

    def texture(self, i):
        if i not in self.tex_map:
            src = self.reader.gltf["textures"][i]
            tex = {k: v for k, v in src.items() if k not in ("sampler", "source", "extensions")}
            if "sampler" in src:
                s = src["sampler"]
                if s not in self.smp_map:
                    self.smp_map[s] = len(self.out.samplers)
                    self.out.samplers.append(copy.deepcopy(self.reader.gltf["samplers"][s]))
                tex["sampler"] = self.smp_map[s]
            if "source" in src:
                tex["source"] = self.image(src["source"])
            self.tex_map[i] = len(self.out.textures)
            self.out.textures.append(tex)
        return self.tex_map[i]

    def material(self, i) -> dict:
        """A copy of material i with every textureInfo (`...Texture: {"index": i}`) re-indexed."""
        def remap(obj):
            if isinstance(obj, dict):
                for k, v in obj.items():
                    if k.endswith("Texture") and isinstance(v, dict) and "index" in v:
                        v["index"] = self.texture(v["index"])
                    remap(v)
            elif isinstance(obj, list):
                for v in obj:
                    remap(v)

        mat = copy.deepcopy(self.reader.gltf["materials"][i])
        remap(mat)
        return mat


def _visual(reader: _Reader, prim: dict) -> Optional[GltfVisual]:
    """TEXCOORD_0, the material and what it references, re-indexed from 0; None when the primitive has neither."""
    uv_acc = prim["attributes"].get("TEXCOORD_0")
    if uv_acc is None and "material" not in prim:
        return None
    vis = GltfVisual()
    if uv_acc is not None:
        vis.uv = reader.float_accessor(uv_acc).astype(np.float32)
    if "material" not in prim:
        return vis
    vis.material = _Collector(reader, vis).material(prim["material"])
    return vis


def _multi_visual(reader: _Reader, prims: list, n_verts: list, n_faces: list) -> GltfMultiVisual:
    """The `GltfMultiVisual` of the included primitives `prims` with their vertex and face counts."""
    ends_v, ends_f = np.cumsum(n_verts), np.cumsum(n_faces)
    vis = GltfMultiVisual(vertex_ranges=np.stack([ends_v - n_verts, n_verts], 1).astype(np.int64),
                          face_ranges=np.stack([ends_f - n_faces, n_faces], 1).astype(np.int64),
                          has_uv=np.array(["TEXCOORD_0" in p["attributes"] for p in prims]))
    if vis.has_uv.any():
        vis.uv = np.zeros((int(ends_v[-1]), 2), np.float32)
        for p, (start, count) in zip(prims, vis.vertex_ranges):
            if "TEXCOORD_0" in p["attributes"]:
                uv = reader.float_accessor(p["attributes"]["TEXCOORD_0"]).astype(np.float32)
                if uv.shape != (count, 2):
                    raise ValueError(f"{reader.path}: a TEXCOORD_0 of shape {uv.shape} on a primitive of {count} vertices")
                vis.uv[start:start + count] = uv
    collector, mat_map = _Collector(reader, vis), {}
    for p in prims:
        m = p.get("material")
        if m is not None and m not in mat_map:
            mat_map[m] = len(vis.materials)
            vis.materials.append(collector.material(m))
        vis.primitive_material.append(None if m is None else mat_map[m])
    return vis


def _mime_type(data: bytes) -> str:
    if data[:8] == b"\x89PNG\r\n\x1a\n":
        return "image/png"
    if data[:3] == b"\xff\xd8\xff":
        return "image/jpeg"
    if data[:4] == b"RIFF" and data[8:12] == b"WEBP":
        return "image/webp"
    raise ValueError("image of unknown type (neither PNG, JPEG nor WebP)")


@dataclass
class _Primitive:
    """One primitive `load_glb` includes: its mesh, node, node world matrix and JSON, POSITION as stored (float64), the
    vertices in world space and its triangles (reversed where the world matrix mirrors)."""
    mesh: int
    node: int
    world: np.ndarray
    prim: dict
    positions: np.ndarray
    vertices: np.ndarray
    triangles: np.ndarray


def _included_primitives(gltf: dict, reader: _Reader, path, visited: Optional[dict] = None) -> list:
    """The triangle primitives `load_glb` includes, in its order (`visited` as in `_mesh_instances`)."""
    out = []
    for mesh_i, world, node in _mesh_instances(gltf, path, visited):
        for prim in gltf["meshes"][mesh_i]["primitives"]:
            mode = prim.get("mode", TRIANGLES)
            if mode not in (TRIANGLES, TRIANGLE_STRIP, TRIANGLE_FAN) or "POSITION" not in prim["attributes"]:
                continue
            pos = reader.float_accessor(prim["attributes"]["POSITION"])
            idx = (reader.accessor(prim["indices"])[:, 0].astype(np.int64) if "indices" in prim
                   else np.arange(len(pos), dtype=np.int64))
            if len(idx) and (idx.min() < 0 or idx.max() >= len(pos)):
                raise ValueError(f"{path}: mesh {mesh_i} has an index outside its {len(pos)} vertices")
            tri = _triangles(idx, mode)
            if not len(tri):
                continue
            if np.linalg.det(world[:3, :3]) < 0:
                tri = tri[:, ::-1]
            out.append(_Primitive(mesh_i, node, world, prim, pos, pos @ world[:3, :3].T + world[:3, 3], tri))
    return out


def load_glb(path) -> Mesh:
    """Read a .glb file into one `Mesh`: the reference's `load_glb` (trimesh `load(..., force="mesh")`).

    Every triangle primitive (modes 4, 5 and 6; strips and fans triangulated as glTF defines) of every mesh node reachable
    from the default scene is included, in depth-first node order and then primitive order; a mesh used by two nodes
    appears twice.  POSITION is transformed by the node's world matrix (parent -> child, float64); where that matrix
    mirrors (negative determinant) the triangles are reversed so that every face stays counter-clockwise.  Points and
    lines are skipped.  Vertices float64 (V, 3), faces int64 (F, 3).

    Vertices are returned as stored: trimesh's load-time merge of duplicate vertices is not restated.  The mesh-input
    pipeline merges them itself (`mesh_input.merge_and_clean_mesh`) and expands its outputs back to these vertices.

    When the geometry is exactly one primitive with TEXCOORD_0 and/or a material, `visual` is a `GltfVisual` (UVs,
    material, textures, samplers, image bytes).  With several included primitives, at least one of them with TEXCOORD_0
    or a material, it is a `GltfMultiVisual`: each primitive's vertex and face range, UVs and material.  Otherwise None.

    ValueError: no triangles, an extension in `extensionsRequired`, a sparse accessor, a bad GLB header or chunk layout."""
    data = Path(path).read_bytes()
    gltf, binary = _parse_glb(data, path)
    required = gltf.get("extensionsRequired") or []
    if required:
        raise ValueError(f"{path}: required glTF extension(s) not supported: {', '.join(required)}")
    reader = _Reader(gltf, binary, path)
    included = _included_primitives(gltf, reader, path)
    verts, faces, prims, n, n_verts, n_faces = [], [], [], 0, [], []
    for p in included:
        verts.append(p.vertices)
        faces.append(p.triangles + n)
        prims.append(p.prim)
        n_verts.append(len(p.vertices))
        n_faces.append(len(p.triangles))
        n += len(p.vertices)
    if not faces:
        raise ValueError(f"No mesh geometry found in {path}")
    visual = None
    if len(prims) == 1:
        visual = _visual(reader, prims[0])
    elif any("TEXCOORD_0" in p["attributes"] or "material" in p for p in prims):
        visual = _multi_visual(reader, prims, np.array(n_verts), np.array(n_faces))
    return Mesh(vertices=np.concatenate(verts), faces=np.ascontiguousarray(np.concatenate(faces)), visual=visual)


# --------------------------------------------------------------------------------------------------------------- the rig
MAX_RIG_JOINTS = 1024
MAX_INFLUENCES = 8
RIG_TOLERANCE = 1e-6         # a parent's world matrix is a rotation times a uniform scale to this relative tolerance
BIND_TOLERANCE = 1e-5        # the default pose reproduces the rest vertices to this fraction of the bounding-box diagonal


@dataclass
class GltfRig:
    """The skeleton and skin of a rigged GLB, as `load_rig` reads them (DESIGN.md §21).  Joints are in the skin's order.

    joint_nodes: (J,) the joints' node indices; parent: (J,) int64, the parent joint or -1; order: (J,) a topological
    order (depth-first from the roots, parents first, siblings in skin order); translation / rotation (x, y, z, w) / scale:
    (J, 3) / (J, 4) / (J, 3) fp64, each joint's default local TRS; from_matrix: (J,) bool, joints stored as `matrix`;
    above: (J, 4, 4), the fixed world matrix above each root joint (identity for the others); inverse_bind: (J, 4, 4).
    rest: (V, 3), `load_glb(path).vertices`; points: (V, 3), the positions the binds act on (POSITION for skinned and
    rigid-child vertices, rest for static ones); binds: (NB, 4, 4), the J inverse bind matrices then one effective bind
    (G_k^0)^-1 NodeWorld^0 per rigid-child node; bind_joint: (NB,); slot_bind (V, 8) int32 and slot_weight (V, 8) fp64, used
    slots (weight > 0) first, each row summing to 1 (all zero for a static vertex)."""
    joint_nodes: list
    parent: np.ndarray
    order: np.ndarray
    translation: np.ndarray
    rotation: np.ndarray
    scale: np.ndarray
    from_matrix: np.ndarray
    above: np.ndarray
    inverse_bind: np.ndarray
    rest: np.ndarray
    points: np.ndarray
    binds: np.ndarray
    bind_joint: np.ndarray
    slot_bind: np.ndarray
    slot_weight: np.ndarray


def _similarity_scale(m: np.ndarray) -> Optional[float]:
    """s when the 3x3 `m` is a rotation times the positive uniform scale s (to RIG_TOLERANCE), else None."""
    g = m.T @ m
    s2 = np.trace(g) / 3
    if not s2 > 0 or np.linalg.det(m) <= 0 or np.abs(g - s2 * np.eye(3)).max() > RIG_TOLERANCE * s2:
        return None
    return float(np.sqrt(s2))


def _trs(node: dict, path, name: str) -> tuple:
    """A node's local (translation, rotation (x, y, z, w) unit, scale); a `matrix` is decomposed, ValueError on shear or a
    non-positive scale."""
    if "matrix" not in node:
        q = np.asarray(node.get("rotation", [0.0, 0.0, 0.0, 1.0]), np.float64)
        n = np.linalg.norm(q)
        return (np.asarray(node.get("translation", [0.0, 0.0, 0.0]), np.float64),
                q / n if n > 0 else np.array([0.0, 0.0, 0.0, 1.0]), np.asarray(node.get("scale", [1.0, 1.0, 1.0]), np.float64))
    m = _node_matrix(node)
    if np.abs(m[3] - [0, 0, 0, 1]).max() > 0:
        raise ValueError(f"{path}: {name}'s matrix is not affine")
    lin = m[:3, :3]
    scale = np.linalg.norm(lin, axis=0)
    if np.linalg.det(lin) <= 0 or not (scale > 0).all():
        raise ValueError(f"{path}: {name}'s matrix has a non-positive scale")
    rot = lin / scale
    if np.abs(rot.T @ rot - np.eye(3)).max() > RIG_TOLERANCE:
        raise ValueError(f"{path}: {name}'s matrix has shear")
    return m[:3, 3].copy(), _quaternions(rot), scale


def load_rig(path) -> GltfRig:
    """Read the skeleton and skin of a rigged .glb, with the vertices in `load_glb`'s order -> GltfRig.

    The file is traversed as `load_glb` traverses it.  A skinned primitive's slots come from JOINTS_0/1 (u8 or u16) and
    WEIGHTS_0/1 (float, or normalized u8/u16), each row divided by its fp64 sum, weight-0 slots unused.  A primitive
    without a skin whose node is, or is under, a joint follows its nearest such joint k rigidly (weight 1, bind
    (G_k^0)^-1 NodeWorld^0); any other primitive is static.

    ValueError, saying why: no skin; two distinct skins among the included nodes; a skinned mesh instanced by two nodes;
    more than 1024 joints, a joint outside the default scene or a non-joint node between two joints; a joint `matrix` with
    shear or a non-positive scale; a joint whose parent's default world matrix is not a rotation times a positive uniform
    scale; more than 8 influences per vertex, a row of weights summing to 0 or a used slot's joint outside the skin; morph
    targets with non-zero default weights on a skinned mesh; a buffer that is an external file, or no BIN chunk; a
    default pose that moves a vertex by more than 1e-5 of the rest bounding-box diagonal (glTF skins ignore the skinned
    node's transform, `load_glb` applies it)."""
    data = Path(path).read_bytes()
    gltf, binary = _parse_glb(data, path)
    required = gltf.get("extensionsRequired") or []
    if required:
        raise ValueError(f"{path}: required glTF extension(s) not supported: {', '.join(required)}")
    buffers = gltf.get("buffers") or []
    if binary is None or not buffers or "uri" in buffers[0]:
        raise ValueError(f"{path}: a rig is read from a GLB whose buffer 0 is its BIN chunk")
    if any(not str(b.get("uri", "data:")).startswith("data:") for b in buffers):
        raise ValueError(f"{path}: a buffer is an external file")
    reader = _Reader(gltf, binary, path)
    visited: dict = {}
    included = _included_primitives(gltf, reader, path, visited)
    if not included:
        raise ValueError(f"No mesh geometry found in {path}")
    nodes = gltf.get("nodes", [])
    skins = sorted({nodes[p.node]["skin"] for p in included if "skin" in nodes[p.node]})
    if not skins:
        raise ValueError(f"{path}: no included mesh node has a skin")
    if len(skins) > 1:
        raise ValueError(f"{path}: the included nodes use {len(skins)} distinct skins {skins}; one is supported")
    skin = gltf["skins"][skins[0]]
    instances = {}
    for mesh_i, _, node in _mesh_instances(gltf, path):
        instances.setdefault(mesh_i, set()).add(node)
    for p in included:
        if "skin" in nodes[p.node] and len(instances[p.mesh]) > 1:
            raise ValueError(f"{path}: skinned mesh {p.mesh} is instanced by {len(instances[p.mesh])} nodes")

    joint_nodes = [int(n) for n in skin["joints"]]
    J = len(joint_nodes)
    if not 1 <= J <= MAX_RIG_JOINTS or len(set(joint_nodes)) != J:
        raise ValueError(f"{path}: the skin has {J} joints (distinct, between 1 and {MAX_RIG_JOINTS} supported)")
    index = {n: j for j, n in enumerate(joint_nodes)}
    for n in joint_nodes:
        if n not in visited:
            raise ValueError(f"{path}: joint node {n} is not in the default scene")

    def joint_ancestor(n):
        """(nearest joint among n's strict ancestors or -1, the node directly above n)"""
        up = visited[n][0]
        while up >= 0 and up not in index:
            up = visited[up][0]
        return (index[up] if up >= 0 else -1), visited[n][0]

    parent = np.full(J, -1, np.int64)
    above = np.tile(np.eye(4), (J, 1, 1))
    for j, n in enumerate(joint_nodes):
        k, direct = joint_ancestor(n)
        if k >= 0 and direct != joint_nodes[k]:
            raise ValueError(f"{path}: non-joint node {direct} lies between joints {joint_nodes[k]} and {n}")
        parent[j] = k
        if k < 0 and direct >= 0:
            above[j] = visited[direct][1]
    trs = [_trs(nodes[n], path, f"joint node {n}") for n in joint_nodes]
    translation = np.stack([t[0] for t in trs])
    rotation = np.stack([t[1] for t in trs])
    scale = np.stack([t[2] for t in trs])
    world0 = np.stack([visited[n][1] for n in joint_nodes])
    for j in range(J):
        pw = world0[parent[j]] if parent[j] >= 0 else above[j]
        if _similarity_scale(pw[:3, :3]) is None:
            raise ValueError(f"{path}: the parent of joint node {joint_nodes[j]} is not a rotation times a positive uniform "
                             "scale at the default pose")
    children = [[] for _ in range(J)]
    for j in range(J):
        if parent[j] >= 0:
            children[parent[j]].append(j)
    order, stack = [], [j for j in range(J - 1, -1, -1) if parent[j] < 0]
    while stack:
        j = stack.pop()
        order.append(j)
        stack.extend(reversed(children[j]))
    if "inverseBindMatrices" in skin:
        ibm = reader.float_accessor(skin["inverseBindMatrices"])
        if ibm.shape != (J, 16):
            raise ValueError(f"{path}: inverseBindMatrices has shape {ibm.shape}, expected ({J}, 16)")
        ibm = ibm.reshape(J, 4, 4).transpose(0, 2, 1)
    else:
        ibm = np.tile(np.eye(4), (J, 1, 1))

    binds, bind_joint, rigid = list(ibm), list(range(J)), {}
    points, slot_bind, slot_weight = [], [], []
    for p in included:
        node, nv = nodes[p.node], len(p.vertices)
        sb, sw = np.zeros((nv, MAX_INFLUENCES), np.int32), np.zeros((nv, MAX_INFLUENCES))
        attrs = p.prim["attributes"]
        if "skin" in node:
            if p.prim.get("targets") and np.any(np.asarray(node.get("weights", gltf["meshes"][p.mesh].get("weights", []))) != 0):
                raise ValueError(f"{path}: skinned mesh {p.mesh} has morph targets with non-zero default weights")
            if any(k.startswith(("JOINTS_", "WEIGHTS_")) and k not in ("JOINTS_0", "JOINTS_1", "WEIGHTS_0", "WEIGHTS_1")
                   for k in attrs):
                raise ValueError(f"{path}: mesh {p.mesh} has more than {MAX_INFLUENCES} influences per vertex")
            sets = [s for s in ("0", "1") if "JOINTS_" + s in attrs or "WEIGHTS_" + s in attrs]
            if "0" not in sets or any("JOINTS_" + s not in attrs or "WEIGHTS_" + s not in attrs for s in sets):
                raise ValueError(f"{path}: skinned mesh {p.mesh} lacks a JOINTS_n / WEIGHTS_n pair")
            jnt = np.concatenate([reader.accessor(attrs["JOINTS_" + s]) for s in sets], 1)
            wgt = np.concatenate([reader.float_accessor(attrs["WEIGHTS_" + s]) for s in sets], 1)
            if jnt.dtype.kind != "u" or jnt.dtype.itemsize > 2 or jnt.shape != (nv, 4 * len(sets)) or wgt.shape != jnt.shape:
                raise ValueError(f"{path}: mesh {p.mesh}'s JOINTS_n / WEIGHTS_n are not u8/u16 and float/normalized VEC4s "
                                 f"over its {nv} vertices")
            total = wgt.sum(1, keepdims=True)
            if not (total > 0).all():
                raise ValueError(f"{path}: mesh {p.mesh} has a vertex whose weights sum to 0")
            wgt = wgt / total
            used = wgt > 0
            if (jnt[used] >= J).any():
                raise ValueError(f"{path}: mesh {p.mesh} has a joint index outside the skin's {J} joints")
            rank = np.argsort(~used, axis=1, kind="stable")       # used slots first, each group in slot order
            k = used.sum(1, keepdims=True)
            live = np.arange(jnt.shape[1])[None] < k
            sb[:, :jnt.shape[1]] = np.where(live, np.take_along_axis(jnt, rank, 1), 0)
            sw[:, :jnt.shape[1]] = np.where(live, np.take_along_axis(wgt, rank, 1), 0.0)
            points.append(p.positions)
        else:
            k = index[p.node] if p.node in index else joint_ancestor(p.node)[0]
            if k >= 0:
                if p.node not in rigid:
                    rigid[p.node] = len(binds)
                    binds.append(np.linalg.inv(world0[k]) @ p.world)
                    bind_joint.append(k)
                sb[:, 0], sw[:, 0] = rigid[p.node], 1.0
                points.append(p.positions)
            else:
                points.append(p.vertices)
        slot_bind.append(sb)
        slot_weight.append(sw)
    rest = np.concatenate([p.vertices for p in included])
    rig = GltfRig(joint_nodes=joint_nodes, parent=parent, order=np.array(order, np.int64), translation=translation,
                  rotation=rotation, scale=scale, from_matrix=np.array(["matrix" in nodes[n] for n in joint_nodes]),
                  above=above, inverse_bind=ibm, rest=rest, points=np.concatenate(points), binds=np.stack(binds),
                  bind_joint=np.array(bind_joint, np.int64), slot_bind=np.concatenate(slot_bind),
                  slot_weight=np.concatenate(slot_weight))
    posed = rig_pose(rig, world0)
    diag = float(np.linalg.norm(rest.max(0) - rest.min(0)))
    err = float(np.abs(posed - rest).max()) if len(rest) else 0.0
    if err > BIND_TOLERANCE * max(diag, np.finfo(float).tiny):
        raise ValueError(f"{path}: the default pose is not the bind pose: it moves a vertex by {err:.3e}, more than "
                         f"{BIND_TOLERANCE:g} of the rest bounding-box diagonal {diag:.3e}")
    return rig


def rig_pose(rig: GltfRig, joint_world: np.ndarray) -> np.ndarray:
    """(V, 3) vertices of `rig` for the (J, 4, 4) joint world matrices, by plain float64 linear blend skinning (static
    vertices at rest)."""
    skin = np.einsum("bij,bjk->bik", joint_world[rig.bind_joint], rig.binds)
    out = np.zeros_like(rig.rest)
    for k in range(MAX_INFLUENCES):
        m = skin[rig.slot_bind[:, k]]
        out += rig.slot_weight[:, k:k + 1] * (np.einsum("vij,vj->vi", m[:, :3, :3], rig.points) + m[:, :3, 3])
    static = ~(rig.slot_weight[:, 0] > 0)
    out[static] = rig.rest[static]
    return out


# ------------------------------------------------------------------------------------------------------------------ writing
class _GlbBuilder:
    """One BIN buffer plus the bufferViews and accessors that index it."""

    def __init__(self):
        self.bin = bytearray()
        self.views: list = []
        self.accessors: list = []

    def view(self, data: bytes, target: Optional[int] = None) -> int:
        self.bin += b"\0" * ((-len(self.bin)) % 4)
        v = {"buffer": 0, "byteOffset": len(self.bin), "byteLength": len(data)}
        if target is not None:
            v["target"] = target
        self.bin += data
        self.views.append(v)
        return len(self.views) - 1

    def accessor(self, arr: np.ndarray, component: int, type_: str, target: Optional[int] = None,
                 min_max: bool = False) -> int:
        arr = np.ascontiguousarray(arr, dtype=COMPONENT_DTYPES[component])
        acc = {"bufferView": self.view(arr.tobytes(), target), "componentType": component,
               "count": int(arr.shape[0]), "type": type_}
        if min_max:
            flat = arr.reshape(arr.shape[0], -1)
            acc["min"], acc["max"] = flat.min(0).tolist(), flat.max(0).tolist()
        self.accessors.append(acc)
        return len(self.accessors) - 1

    def add_visual(self, gltf: dict, attributes: dict, visual: Optional[GltfVisual], n_vertices: int) -> None:
        """TEXCOORD_0 into `attributes`; material, textures, samplers and images into `gltf`."""
        if visual is None:
            return
        if visual.uv is not None:
            uv = np.asarray(visual.uv, dtype=np.float32)
            if uv.shape != (n_vertices, 2):
                raise ValueError(f"visual.uv has shape {uv.shape}, expected ({n_vertices}, 2)")
            attributes["TEXCOORD_0"] = self.accessor(uv, F32, "VEC2", ARRAY_BUFFER)
        if visual.material is not None:
            gltf["materials"] = [copy.deepcopy(visual.material)]
        for key in ("textures", "samplers"):
            if getattr(visual, key):
                gltf[key] = copy.deepcopy(getattr(visual, key))
        if visual.images:
            gltf["images"] = [{**img, "bufferView": self.view(bytes(data))}
                              for img, data in zip(visual.images, visual.image_bytes)]

    def add_primitives(self, gltf: dict, visual: GltfMultiVisual, faces: np.ndarray, per_vertex: list,
                       targets: Optional[np.ndarray] = None, default_material: bool = True) -> list:
        """One triangle primitive per range of `visual` (checked by the caller) -> the primitives.  Primitive p gets the
        rows of its vertex range of every (name, array, component, type, min_max) in `per_vertex`, TEXCOORD_0 when
        has_uv[p], its faces rebased to its range as u32 indices, its material (the default blue when it has none and
        `default_material`) and the rows of its range of each (T, V, 3) morph target.  Materials, textures, samplers and
        images go into `gltf`."""
        materials, default, prims = copy.deepcopy(visual.materials), None, []
        for p, ((v0, nv), (f0, nf)) in enumerate(zip(np.asarray(visual.vertex_ranges), np.asarray(visual.face_ranges))):
            rows = slice(int(v0), int(v0 + nv))
            attributes = {name: self.accessor(arr[rows], comp, type_, ARRAY_BUFFER, min_max=mm)
                          for name, arr, comp, type_, mm in per_vertex}
            if visual.has_uv[p]:
                attributes["TEXCOORD_0"] = self.accessor(np.asarray(visual.uv, np.float32)[rows], F32, "VEC2", ARRAY_BUFFER)
            prim = {"attributes": attributes,
                    "indices": self.accessor((faces[f0:f0 + nf] - v0).reshape(-1, 1), U32, "SCALAR", ELEMENT_ARRAY_BUFFER)}
            material = visual.primitive_material[p]
            if material is None and default_material:
                if default is None:
                    default = len(materials)
                    materials.append(copy.deepcopy(DEFAULT_MATERIAL))
                material = default
            if material is not None:
                prim["material"] = int(material)
            prim["mode"] = TRIANGLES
            if targets is not None:
                prim["targets"] = [{"POSITION": self.accessor(t[rows], F32, "VEC3", ARRAY_BUFFER, min_max=True)}
                                   for t in targets]
            prims.append(prim)
        if materials:
            gltf["materials"] = materials
        for key in ("textures", "samplers"):
            if getattr(visual, key):
                gltf[key] = copy.deepcopy(getattr(visual, key))
        if visual.images:
            gltf["images"] = [{**img, "bufferView": self.view(bytes(data))}
                              for img, data in zip(visual.images, visual.image_bytes)]
        return prims

    def write(self, path, gltf: dict) -> None:
        gltf = {"asset": {"version": "2.0", "generator": "actionmesh_b200"}, **gltf}
        if self.bin:
            self.bin += b"\0" * ((-len(self.bin)) % 4)
            gltf["buffers"] = [{"byteLength": len(self.bin)}]
            gltf["bufferViews"] = self.views
            gltf["accessors"] = self.accessors
        js = json.dumps(gltf, separators=(",", ":")).encode("utf-8")
        js += b" " * ((-len(js)) % 4)
        chunks = struct.pack("<II", len(js), CHUNK_JSON) + js
        if self.bin:
            chunks += struct.pack("<II", len(self.bin), CHUNK_BIN) + bytes(self.bin)
        with open(path, "wb") as f:
            f.write(GLB_MAGIC + struct.pack("<II", 2, 12 + len(chunks)) + chunks)


def _mesh_arrays(mesh) -> tuple[np.ndarray, np.ndarray]:
    return np.asarray(mesh.vertices), np.asarray(mesh.faces).reshape(-1, 3)


def _check_faces(faces: np.ndarray, n_vertices: int) -> None:
    if len(faces) and (faces.min() < 0 or faces.max() >= n_vertices):
        raise ValueError(f"faces index outside the {n_vertices} vertices")


def write_glb(path, mesh) -> None:
    """Write `mesh` (`.vertices` (V, 3), `.faces` (F, 3)) as a GLB file: one scene, one node, one mesh, one triangle
    primitive, what trimesh exports for an untextured `Trimesh(process=False)`.  POSITION is float32 with min/max, indices
    u32.  A `GltfVisual` in `mesh.visual` is written as TEXCOORD_0 plus its material, textures, samplers and images.  A
    `GltfMultiVisual` gives one primitive per range instead, each with its own POSITION, TEXCOORD_0 (when it has UVs),
    rebased indices and material (none when it has none); ValueError when its ranges do not fit the mesh.  A mesh without
    faces gives a scene whose one node has no mesh."""
    verts, faces = _mesh_arrays(mesh)
    _check_faces(faces, len(verts))
    b = _GlbBuilder()
    gltf: dict = {"scene": 0, "scenes": [{"nodes": [0]}], "nodes": [{}]}
    visual = getattr(mesh, "visual", None)
    if len(faces) and isinstance(visual, GltfMultiVisual):
        check_multi_visual(visual, len(verts), faces)
        prims = b.add_primitives(gltf, visual, faces, [("POSITION", np.asarray(verts, np.float32), F32, "VEC3", True)],
                                 default_material=False)
        gltf["meshes"] = [{"primitives": prims}]
        gltf["nodes"] = [{"mesh": 0}]
    elif len(faces):
        attributes = {"POSITION": b.accessor(verts, F32, "VEC3", ARRAY_BUFFER, min_max=True)}
        prim = {"attributes": attributes, "indices": b.accessor(faces.reshape(-1, 1), U32, "SCALAR",
                                                                ELEMENT_ARRAY_BUFFER), "mode": TRIANGLES}
        visual = getattr(mesh, "visual", None)
        b.add_visual(gltf, attributes, visual if isinstance(visual, GltfVisual) else None, len(verts))
        if "materials" in gltf:
            prim["material"] = 0
        gltf["meshes"] = [{"primitives": [prim]}]
        gltf["nodes"] = [{"mesh": 0}]
    b.write(path, gltf)


def write_animated_glb(path, vertices, faces, fps: float = 8, visual=None) -> None:
    """Write (T, V, 3) `vertices` on (F, 3) `faces` as an animated GLB: the file the reference's `create_animated_glb`
    gets from Blender, without Blender.

    One morph target per frame (POSITION deltas, float32 with min/max; the mesh's `extras.targetNames` are Frame_0 ...)
    and one LINEAR `weights` animation with keyframes at k / fps whose weights are the T x T identity: frame k shows
    target k alone.  Positions are mapped by `ANIMATED_GLB_MAP` as the reference's npy + Blender export maps them: the base
    is M v_0 and target k holds M v_k - M v_0.  Without `visual` the material is the reference's default blue,
    double-sided; with one its UVs, material and textures are kept.  A `GltfMultiVisual` gives one primitive per range,
    each with the T targets over its range and its own material (the default blue when it has none).  No normals, no Draco: about 12 T V bytes of morph
    data (7 MB at 31 frames x 20 000 vertices)."""
    v = np.asarray(vertices, dtype=np.float64)
    f = np.asarray(faces).reshape(-1, 3)
    if v.ndim != 3 or v.shape[0] < 1 or v.shape[2] != 3:
        raise ValueError(f"vertices must be (T, V, 3) with T >= 1, got {v.shape}")
    if not len(f):
        raise ValueError("an animated GLB needs at least one face")
    _check_faces(f, v.shape[1])
    n_frames = v.shape[0]
    mapped = v @ ANIMATED_GLB_MAP.T
    base = mapped[0].astype(np.float32)
    b = _GlbBuilder()
    gltf: dict = {"scene": 0, "scenes": [{"nodes": [0]}], "nodes": [{"mesh": 0, "name": "AnimatedMesh"}]}
    weights = np.eye(n_frames, dtype=np.float32)
    mesh = {"name": "AnimatedMesh", "weights": weights[0].tolist(),
            "extras": {"targetNames": [f"Frame_{k}" for k in range(n_frames)]}}
    if isinstance(visual, GltfMultiVisual):
        check_multi_visual(visual, v.shape[1], f)
        targets = (mapped - base).astype(np.float32)
        mesh["primitives"] = b.add_primitives(gltf, visual, f, [("POSITION", base, F32, "VEC3", True)], targets)
        gltf["meshes"] = [mesh]
        _write_weights_animation(b, gltf, weights, fps)
        b.write(path, gltf)
        return
    attributes = {"POSITION": b.accessor(base, F32, "VEC3", ARRAY_BUFFER, min_max=True)}
    targets = [{"POSITION": b.accessor((mapped[k] - base).astype(np.float32), F32, "VEC3", ARRAY_BUFFER, min_max=True)}
               for k in range(n_frames)]
    indices = b.accessor(f.reshape(-1, 1), U32, "SCALAR", ELEMENT_ARRAY_BUFFER)
    b.add_visual(gltf, attributes, visual, v.shape[1])
    if "materials" not in gltf:
        gltf["materials"] = [copy.deepcopy(DEFAULT_MATERIAL)]
    mesh["primitives"] = [{"attributes": attributes, "indices": indices, "material": 0, "mode": TRIANGLES, "targets": targets}]
    gltf["meshes"] = [mesh]
    _write_weights_animation(b, gltf, weights, fps)
    b.write(path, gltf)


def _write_weights_animation(b: _GlbBuilder, gltf: dict, weights: np.ndarray, fps: float) -> None:
    """The animated GLB's one LINEAR `weights` animation of node 0: keyframe k at k / fps holds row k of `weights`."""
    n_frames = len(weights)
    times = b.accessor((np.arange(n_frames, dtype=np.float64) / fps).astype(np.float32).reshape(-1, 1), F32, "SCALAR",
                       min_max=True)
    gltf["animations"] = [{"name": "Animation",
                           "channels": [{"sampler": 0, "target": {"node": 0, "path": "weights"}}],
                           "samplers": [{"input": times, "output": b.accessor(weights.reshape(-1, 1), F32, "SCALAR"),
                                         "interpolation": "LINEAR"}]}]


def _quaternions(rot: np.ndarray) -> np.ndarray:
    """(..., 3, 3) proper rotations -> (..., 4) unit quaternions (x, y, z, w), glTF's order, from the largest of the four
    squared components (Shepperd's method)."""
    r = np.asarray(rot, dtype=np.float64)
    tr = r[..., 0, 0] + r[..., 1, 1] + r[..., 2, 2]
    sq = np.stack([1 + 2 * r[..., 0, 0] - tr, 1 + 2 * r[..., 1, 1] - tr, 1 + 2 * r[..., 2, 2] - tr, 1 + tr], -1)
    k = np.argmax(sq, -1)
    q = np.empty(r.shape[:-2] + (4,))
    s = np.sqrt(np.maximum(np.take_along_axis(sq, k[..., None], -1)[..., 0], 1e-300))    # 4 |q_k|
    off = {(0, 1): r[..., 0, 1] + r[..., 1, 0], (0, 2): r[..., 0, 2] + r[..., 2, 0], (1, 2): r[..., 1, 2] + r[..., 2, 1],
           (0, 3): r[..., 2, 1] - r[..., 1, 2], (1, 3): r[..., 0, 2] - r[..., 2, 0], (2, 3): r[..., 1, 0] - r[..., 0, 1]}
    for a in range(4):
        sel = k == a
        for b in range(4):
            q[..., b] = np.where(sel, s / 2 if a == b else off[min(a, b), max(a, b)] / (2 * s), q[..., b])
    return q / np.linalg.norm(q, axis=-1, keepdims=True)


def _checked_skin(rest: np.ndarray, faces, joints, weights, n_joints: int, what: str,
                  noun: str) -> tuple[np.ndarray, np.ndarray]:
    """(faces (F, 3), weights divided by their row sums) after the checks every skinned file makes; `what` names the
    file and `noun` its joints in the messages."""
    f = np.asarray(faces).reshape(-1, 3)
    if not len(f):
        raise ValueError(f"{what} needs at least one face")
    _check_faces(f, len(rest))
    j = np.asarray(joints)
    if n_joints > 256 or j.shape != (len(rest), 4) or j.min() < 0 or j.max() >= n_joints:
        raise ValueError(f"joints must be (V, 4) indices of the {n_joints} {noun} (at most 256)")
    w = np.asarray(weights, dtype=np.float64)
    total = w.sum(1, keepdims=True) if w.ndim == 2 else np.zeros(1)
    if w.shape != (len(rest), 4) or (w < 0).any() or not (total > 0).all():
        raise ValueError("weights must be (V, 4), non-negative, with a positive sum per vertex")
    return f, w / total


def _key_quaternions(rot: np.ndarray) -> np.ndarray:
    """(T, J, 3, 3) rotations -> (T, J, 4) quaternions of M R M^T (M = ANIMATED_GLB_MAP), each key's sign chosen so that its
    dot product with the previous key's is >= 0."""
    quat = _quaternions(ANIMATED_GLB_MAP @ rot @ ANIMATED_GLB_MAP.T)
    for k in range(1, len(quat)):
        quat[k] *= np.where((quat[k] * quat[k - 1]).sum(-1) < 0, -1.0, 1.0)[:, None]
    return quat


def _skinned_mesh(b: _GlbBuilder, gltf: dict, rest: np.ndarray, joints, weights: np.ndarray, f: np.ndarray, visual) -> None:
    """gltf["meshes"] = one "SkinnedMesh": POSITION = M p (float32 with min/max), JOINTS_0 (u8), WEIGHTS_0 (float32,
    rows already normalised), with the visual's UVs and material (the default blue without one), or one primitive per
    range of a `GltfMultiVisual`."""
    per_vertex = [("POSITION", (rest @ ANIMATED_GLB_MAP.T).astype(np.float32), F32, "VEC3", True),
                  ("JOINTS_0", np.asarray(joints, dtype=np.uint8), U8, "VEC4", False),
                  ("WEIGHTS_0", weights.astype(np.float32), F32, "VEC4", False)]
    if isinstance(visual, GltfMultiVisual):
        check_multi_visual(visual, len(rest), f)
        gltf["meshes"] = [{"name": "SkinnedMesh", "primitives": b.add_primitives(gltf, visual, f, per_vertex)}]
    else:
        attributes = {name: b.accessor(arr, comp, type_, ARRAY_BUFFER, min_max=mm) for name, arr, comp, type_, mm in per_vertex}
        indices = b.accessor(f.reshape(-1, 1), U32, "SCALAR", ELEMENT_ARRAY_BUFFER)
        b.add_visual(gltf, attributes, visual, len(rest))
        if "materials" not in gltf:
            gltf["materials"] = [copy.deepcopy(DEFAULT_MATERIAL)]
        gltf["meshes"] = [{"name": "SkinnedMesh", "primitives": [{"attributes": attributes, "indices": indices,
                                                                  "material": 0, "mode": TRIANGLES}]}]


def write_skinned_glb(path, fit, faces, fps: float = 8, visual=None) -> None:
    """Write a `skinning.SkinningFit` on (F, 3) `faces` as a skinned GLB: one rest mesh, n_bones joints and one LINEAR
    animation, in the coordinates of `write_animated_glb` (DESIGN §20).

    The mesh node carries skin 0; its primitive has POSITION = M p (float32 with min/max), JOINTS_0 (u8) and WEIGHTS_0
    (float32, each row divided by its sum).  Joint j is a child of the root node "Armature", placed at M c_j (c_j: the bone's
    rest centre), with inverse bind matrix translate(-M c_j).  Keyframe k at k / fps sets joint j's rotation to the
    quaternion of M R_j^k M^T (each key's sign chosen closest to the previous key's) and its translation to
    M (R_j^k c_j + t_j^k), so that the joint matrix is M [R_j^k | t_j^k] M^T.  Without `visual` the material is the animated
    GLB's default blue, double-sided; with one its UVs, material and textures are kept.  A `GltfMultiVisual` gives one
    primitive per range, each with JOINTS_0 and WEIGHTS_0 over its range under the one skin and its own material (the
    default blue when it has none)."""
    rest = np.asarray(fit.rest, dtype=np.float64)
    rot, trans, centres = (np.asarray(a, dtype=np.float64) for a in (fit.rotations, fit.translations, fit.centres))
    T, B = rot.shape[:2]
    f, w = _checked_skin(rest, faces, fit.joints, fit.weights, B, "a skinned GLB", "bones")
    M = ANIMATED_GLB_MAP
    mc = centres @ M.T
    joint_nodes = list(range(2, 2 + B))
    gltf: dict = {"scene": 0, "scenes": [{"nodes": [0, 1]}],
                  "nodes": [{"mesh": 0, "skin": 0, "name": "SkinnedMesh"}, {"name": "Armature", "children": joint_nodes}]
                  + [{"name": f"Bone_{j}", "translation": mc[j].tolist()} for j in range(B)]}
    b = _GlbBuilder()
    _skinned_mesh(b, gltf, rest, fit.joints, w, f, visual)
    ibm = np.tile(np.eye(4), (B, 1, 1))
    ibm[:, :3, 3] = -mc
    gltf["skins"] = [{"joints": joint_nodes, "skeleton": 1,
                      "inverseBindMatrices": b.accessor(ibm.transpose(0, 2, 1).reshape(B, 16).astype(np.float32), F32,
                                                        "MAT4")}]
    quat = _key_quaternions(rot)                                                         # (T, B, 4)
    node_t = (np.einsum("tbij,bj->tbi", rot, centres) + trans) @ M.T                    # (T, B, 3)
    times = b.accessor((np.arange(T, dtype=np.float64) / fps).astype(np.float32).reshape(-1, 1), F32, "SCALAR",
                       min_max=True)
    samplers, channels = [], []
    for j in range(B):
        for path_, data, type_ in (("translation", node_t[:, j], "VEC3"), ("rotation", quat[:, j], "VEC4")):
            samplers.append({"input": times, "output": b.accessor(data.astype(np.float32), F32, type_),
                             "interpolation": "LINEAR"})
            channels.append({"sampler": len(samplers) - 1, "target": {"node": joint_nodes[j], "path": path_}})
    gltf["animations"] = [{"name": "Animation", "channels": channels, "samplers": samplers}]
    b.write(path, gltf)


def write_auto_rig_glb(path, fit, faces, fps: float = 8, visual=None) -> None:
    """Write an `autorig.AutoRigFit` on (F, 3) `faces` as a rigged GLB in the coordinates of `write_animated_glb`
    (DESIGN §22): the mesh and material as `write_skinned_glb` writes them, and a joint hierarchy "Joint_<k>" nested under
    "Armature" in the fit's depth-first order.

    Joint k's node translation is M (c_k - c_parent) (M c_root for the root), its inverse bind translate(-M c_k).  One
    LINEAR animation keys, at k / fps, every joint's rotation (the quaternion of M R M^T, each key's sign chosen closest
    to the previous key's) and the root's translation M tau.  Conjugating by the reflection M keeps every composition, so
    key k shows M v^ of the fit's frame k."""
    rest = np.asarray(fit.rest, dtype=np.float64)
    rot = np.asarray(fit.rotation_matrices, dtype=np.float64)
    T, J = rot.shape[:2]
    parent = np.asarray(fit.parent, np.int64)
    f, w = _checked_skin(rest, faces, fit.joints, fit.weights, J, "a rigged GLB", "joints")
    if parent.shape != (J,) or parent[0] != -1 or (parent[1:] < 0).any() or (parent[1:] >= np.arange(1, J)).any():
        raise ValueError("parent must list a depth-first tree rooted at joint 0")
    M = ANIMATED_GLB_MAP
    mc = np.asarray(fit.positions, dtype=np.float64) @ M.T
    joint_nodes = list(range(2, 2 + J))
    nodes = [{"mesh": 0, "skin": 0, "name": "RiggedMesh"}, {"name": "Armature", "children": [2]}]
    for k in range(J):
        node = {"name": f"Joint_{k}", "translation": (mc[k] - mc[parent[k]] if k else mc[k]).tolist()}
        children = [2 + c for c in np.flatnonzero(parent == k)]
        if children:
            node["children"] = [int(c) for c in children]
        nodes.append(node)
    gltf: dict = {"scene": 0, "scenes": [{"nodes": [0, 1]}], "nodes": nodes}
    b = _GlbBuilder()
    _skinned_mesh(b, gltf, rest, fit.joints, w, f, visual)
    ibm = np.tile(np.eye(4), (J, 1, 1))
    ibm[:, :3, 3] = -mc
    gltf["skins"] = [{"joints": joint_nodes, "skeleton": 1,
                      "inverseBindMatrices": b.accessor(ibm.transpose(0, 2, 1).reshape(J, 16).astype(np.float32), F32,
                                                        "MAT4")}]
    quat = _key_quaternions(rot)                                                         # (T, J, 4)
    times = b.accessor((np.arange(T, dtype=np.float64) / fps).astype(np.float32).reshape(-1, 1), F32, "SCALAR",
                       min_max=True)
    samplers = [{"input": times, "output": b.accessor((np.asarray(fit.root_translations) @ M.T).astype(np.float32), F32,
                                                      "VEC3"), "interpolation": "LINEAR"}]
    channels = [{"sampler": 0, "target": {"node": joint_nodes[0], "path": "translation"}}]
    for k in range(J):
        samplers.append({"input": times, "output": b.accessor(quat[:, k].astype(np.float32), F32, "VEC4"),
                         "interpolation": "LINEAR"})
        channels.append({"sampler": len(samplers) - 1, "target": {"node": joint_nodes[k], "path": "rotation"}})
    gltf["animations"] = [{"name": "Animation", "channels": channels, "samplers": samplers}]
    b.write(path, gltf)


def write_rig_animation(src_path, out_path, rig: GltfRig, fit, fps: float = 8) -> None:
    """Write the GLB at `src_path` to `out_path` with a `rig.RigFit` of its `load_rig` rig as a new first animation.

    The JSON and BIN are kept except for: joints stored as `matrix` become their TRS (glTF does not animate `matrix`
    nodes); a LINEAR animation "ActionMesh" inserted as animations[0], with keys at k / fps, a float32 rotation channel
    for every joint (each key's sign chosen so that its dot product with the previous key is >= 0) and a translation
    channel for each root joint; its accessors and bufferViews appended, their data at the end of the BIN chunk (4-byte
    aligned) and buffers[0].byteLength updated.  The file stays in its own frame."""
    gltf, binary = _parse_glb(Path(src_path).read_bytes(), src_path)
    gltf = copy.deepcopy(gltf)
    buffers = gltf.get("buffers") or []
    if binary is None or not buffers or "uri" in buffers[0]:
        raise ValueError(f"{src_path}: the rig animation is written into a GLB whose buffer 0 is its BIN chunk")
    skins_joints = [s["joints"] for s in gltf.get("skins", [])]
    if list(rig.joint_nodes) not in skins_joints:
        raise ValueError(f"{src_path}: the rig's joints are not a skin of this file")
    quat = np.array(fit.rotations, dtype=np.float64)
    trans = np.asarray(fit.translations, dtype=np.float64)
    T, J = quat.shape[:2]
    if J != len(rig.joint_nodes) or quat.shape != (T, J, 4) or trans.shape != (T, J, 3) or T < 1:
        raise ValueError(f"the fit's rotations {quat.shape} and translations {trans.shape} do not match the rig's {len(rig.joint_nodes)} joints")
    for k in range(1, T):
        quat[k] *= np.where((quat[k] * quat[k - 1]).sum(-1) < 0, -1.0, 1.0)[:, None]
    nodes = gltf["nodes"]
    for j, n in enumerate(rig.joint_nodes):
        if "matrix" in nodes[n]:
            del nodes[n]["matrix"]
            nodes[n]["translation"] = rig.translation[j].tolist()
            nodes[n]["rotation"] = rig.rotation[j].tolist()
            nodes[n]["scale"] = rig.scale[j].tolist()
    out = bytearray(binary)
    out += b"\0" * ((-len(out)) % 4)
    views, accessors = gltf.setdefault("bufferViews", []), gltf.setdefault("accessors", [])

    def accessor(arr: np.ndarray, type_: str, min_max: bool = False) -> int:
        arr = np.ascontiguousarray(arr, dtype=np.float32)
        out.extend(b"\0" * ((-len(out)) % 4))
        views.append({"buffer": 0, "byteOffset": len(out), "byteLength": arr.nbytes})
        out.extend(arr.tobytes())
        acc = {"bufferView": len(views) - 1, "componentType": F32, "count": int(arr.shape[0]), "type": type_}
        if min_max:
            acc["min"], acc["max"] = arr.min(0).tolist(), arr.max(0).tolist()
        accessors.append(acc)
        return len(accessors) - 1

    times = accessor((np.arange(T, dtype=np.float64) / fps).reshape(-1, 1), "SCALAR", min_max=True)
    samplers, channels = [], []
    for j, n in enumerate(rig.joint_nodes):
        for path_, data, type_, on in (("rotation", quat[:, j], "VEC4", True),
                                       ("translation", trans[:, j], "VEC3", rig.parent[j] < 0)):
            if on:
                samplers.append({"input": times, "output": accessor(data, type_), "interpolation": "LINEAR"})
                channels.append({"sampler": len(samplers) - 1, "target": {"node": int(n), "path": path_}})
    gltf["animations"] = [{"name": "ActionMesh", "channels": channels, "samplers": samplers}] + gltf.get("animations", [])
    out += b"\0" * ((-len(out)) % 4)
    buffers[0]["byteLength"] = len(out)
    js = json.dumps(gltf, separators=(",", ":")).encode("utf-8")
    js += b" " * ((-len(js)) % 4)
    chunks = struct.pack("<II", len(js), CHUNK_JSON) + js + struct.pack("<II", len(out), CHUNK_BIN) + bytes(out)
    with open(out_path, "wb") as f:
        f.write(GLB_MAGIC + struct.pack("<II", 2, 12 + len(chunks)) + chunks)


# ------------------------------------------------------------------------------------------------------- the reference's IO
def save_deformation(meshes: list, path) -> tuple[Path, Path]:
    """`save_deformation` (actionmesh/io/mesh_io.py:43-102): {stem}_vertices.npy, (T, V, 3) float32 with (x, y, z) ->
    (-z, x, y), and {stem}_faces.npy, (F, 3) int32 -> (vertices path, faces path).  The meshes (trimesh objects or `Mesh`
    records) must share one vertex count and one face array."""
    if len(meshes) == 0:
        raise ValueError("Cannot save deformation from empty mesh list")
    n_verts = len(meshes[0].vertices)
    reference_faces = np.asarray(meshes[0].faces)
    for i, mesh in enumerate(meshes):
        if len(mesh.vertices) != n_verts:
            raise ValueError(f"Mesh {i} has {len(mesh.vertices)} vertices, expected {n_verts} (same as first mesh)")
        faces = np.asarray(mesh.faces)
        if faces.shape != reference_faces.shape or not np.array_equal(faces, reference_faces):
            raise ValueError(f"Mesh {i} has different face topology than the first mesh. "
                             f"All meshes must share the same faces for deformation export.")
    vertices = np.stack([np.asarray(mesh.vertices).astype(np.float32) for mesh in meshes], axis=0)
    vertices = vertices[:, :, [2, 0, 1]]
    vertices[:, :, 0] = -vertices[:, :, 0]
    path = Path(path)
    path.parent.mkdir(parents=True, exist_ok=True)
    vertices_path = path.parent / f"{path.stem}_vertices.npy"
    faces_path = path.parent / f"{path.stem}_faces.npy"
    np.save(vertices_path, vertices)
    np.save(faces_path, reference_faces.astype(np.int32))
    return vertices_path, faces_path


def save_meshes(meshes: list, output_dir) -> list[Path]:
    """`save_meshes` (actionmesh/io/mesh_io.py:105-114): output_dir/mesh_{i:02d}.glb for every mesh, through `write_glb`
    -> the paths."""
    os.makedirs(output_dir, exist_ok=True)
    paths = [Path(output_dir) / f"mesh_{i:02d}.glb" for i in range(len(meshes))]
    for mesh, p in zip(meshes, paths):
        write_glb(p, mesh)
    logger.info(f"Saved {len(meshes)} meshes to {output_dir}")
    return paths
