"""GLB (binary glTF 2.0) files and the deformation arrays, with numpy and the standard library only: the reference's
`actionmesh/io/mesh_io.py` (trimesh) and `actionmesh/io/glb_export.py` (Blender) without either dependency.

  load_glb(path) -> Mesh                     every triangle primitive of the default scene, node transforms applied
  write_glb(path, mesh)                      one node, one mesh, one triangle primitive (what trimesh exports)
  write_animated_glb(path, vertices, faces)  one morph target per frame and a weights animation (what Blender exports)
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
TYPE_SIZES = {"SCALAR": 1, "VEC2": 2, "VEC3": 3, "VEC4": 4}
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


def _mesh_instances(gltf: dict, path) -> list:
    """[(mesh index, 4x4 world transform)] in depth-first node order, children in their listed order."""
    nodes, out = gltf.get("nodes", []), []

    def visit(i, parent, ancestors):
        if i in ancestors:
            raise ValueError(f"{path}: node {i} is its own ancestor")
        world = parent @ _node_matrix(nodes[i])
        if "mesh" in nodes[i]:
            out.append((nodes[i]["mesh"], world))
        for c in nodes[i].get("children", []):
            visit(c, world, ancestors | {i})

    for r in _root_nodes(gltf):
        visit(r, np.eye(4), frozenset())
    return out


def _visual(reader: _Reader, prim: dict) -> Optional[GltfVisual]:
    """TEXCOORD_0, the material and what it references, re-indexed from 0; None when the primitive has neither."""
    gltf = reader.gltf
    uv_acc = prim["attributes"].get("TEXCOORD_0")
    if uv_acc is None and "material" not in prim:
        return None
    vis = GltfVisual()
    if uv_acc is not None:
        vis.uv = reader.float_accessor(uv_acc).astype(np.float32)
    if "material" not in prim:
        return vis
    vis.material = copy.deepcopy(gltf["materials"][prim["material"]])
    tex_map, smp_map, img_map = {}, {}, {}

    def image(i):
        if i not in img_map:
            img = gltf["images"][i]
            data = reader.view_bytes(img["bufferView"]) if "bufferView" in img else _read_uri(img["uri"], reader.path)
            entry = {"mimeType": img.get("mimeType") or _mime_type(data)}
            if "name" in img:
                entry["name"] = img["name"]
            img_map[i] = len(vis.images)
            vis.images.append(entry)
            vis.image_bytes.append(bytes(data))
        return img_map[i]

    def texture(i):
        if i not in tex_map:
            tex = {k: v for k, v in gltf["textures"][i].items() if k not in ("sampler", "source", "extensions")}
            if "sampler" in gltf["textures"][i]:
                s = gltf["textures"][i]["sampler"]
                if s not in smp_map:
                    smp_map[s] = len(vis.samplers)
                    vis.samplers.append(copy.deepcopy(gltf["samplers"][s]))
                tex["sampler"] = smp_map[s]
            if "source" in gltf["textures"][i]:
                tex["source"] = image(gltf["textures"][i]["source"])
            tex_map[i] = len(vis.textures)
            vis.textures.append(tex)
        return tex_map[i]

    def remap(obj):                       # every textureInfo (`...Texture: {"index": i}`) anywhere in the material
        if isinstance(obj, dict):
            for k, v in obj.items():
                if k.endswith("Texture") and isinstance(v, dict) and "index" in v:
                    v["index"] = texture(v["index"])
                remap(v)
        elif isinstance(obj, list):
            for v in obj:
                remap(v)

    remap(vis.material)
    return vis


def _mime_type(data: bytes) -> str:
    if data[:8] == b"\x89PNG\r\n\x1a\n":
        return "image/png"
    if data[:3] == b"\xff\xd8\xff":
        return "image/jpeg"
    if data[:4] == b"RIFF" and data[8:12] == b"WEBP":
        return "image/webp"
    raise ValueError("image of unknown type (neither PNG, JPEG nor WebP)")


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
    material, textures, samplers, image bytes); with several primitives it is None and a warning is logged.

    ValueError: no triangles, an extension in `extensionsRequired`, a sparse accessor, a bad GLB header or chunk layout."""
    data = Path(path).read_bytes()
    gltf, binary = _parse_glb(data, path)
    required = gltf.get("extensionsRequired") or []
    if required:
        raise ValueError(f"{path}: required glTF extension(s) not supported: {', '.join(required)}")
    reader = _Reader(gltf, binary, path)
    verts, faces, prims, n = [], [], [], 0
    for mesh_i, world in _mesh_instances(gltf, path):
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
            verts.append(pos @ world[:3, :3].T + world[:3, 3])
            faces.append(tri + n)
            prims.append(prim)
            n += len(pos)
    if not faces:
        raise ValueError(f"No mesh geometry found in {path}")
    visual = None
    if len(prims) == 1:
        visual = _visual(reader, prims[0])
    elif any("TEXCOORD_0" in p["attributes"] or "material" in p for p in prims):
        logger.warning(f"{path}: {len(prims)} primitives; their UVs and materials are not merged, so the mesh has none")
    return Mesh(vertices=np.concatenate(verts), faces=np.ascontiguousarray(np.concatenate(faces)), visual=visual)


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
    mesh without faces gives a scene whose one node has no mesh."""
    verts, faces = _mesh_arrays(mesh)
    _check_faces(faces, len(verts))
    b = _GlbBuilder()
    gltf: dict = {"scene": 0, "scenes": [{"nodes": [0]}], "nodes": [{}]}
    if len(faces):
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


def write_animated_glb(path, vertices, faces, fps: float = 8, visual: Optional[GltfVisual] = None) -> None:
    """Write (T, V, 3) `vertices` on (F, 3) `faces` as an animated GLB: the file the reference's `create_animated_glb`
    gets from Blender, without Blender.

    One morph target per frame (POSITION deltas, float32 with min/max; the mesh's `extras.targetNames` are Frame_0 ...)
    and one LINEAR `weights` animation with keyframes at k / fps whose weights are the T x T identity: frame k shows
    target k alone.  Positions are mapped by `ANIMATED_GLB_MAP` as the reference's npy + Blender export maps them: the base
    is M v_0 and target k holds M v_k - M v_0.  Without `visual` the material is the reference's default blue,
    double-sided; with one its UVs, material and textures are kept.  No normals, no Draco: about 12 T V bytes of morph
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
    attributes = {"POSITION": b.accessor(base, F32, "VEC3", ARRAY_BUFFER, min_max=True)}
    targets = [{"POSITION": b.accessor((mapped[k] - base).astype(np.float32), F32, "VEC3", ARRAY_BUFFER, min_max=True)}
               for k in range(n_frames)]
    indices = b.accessor(f.reshape(-1, 1), U32, "SCALAR", ELEMENT_ARRAY_BUFFER)
    gltf: dict = {"scene": 0, "scenes": [{"nodes": [0]}], "nodes": [{"mesh": 0, "name": "AnimatedMesh"}]}
    b.add_visual(gltf, attributes, visual, v.shape[1])
    if "materials" not in gltf:
        gltf["materials"] = [copy.deepcopy(DEFAULT_MATERIAL)]
    weights = np.eye(n_frames, dtype=np.float32)
    gltf["meshes"] = [{"name": "AnimatedMesh", "weights": weights[0].tolist(),
                       "extras": {"targetNames": [f"Frame_{k}" for k in range(n_frames)]},
                       "primitives": [{"attributes": attributes, "indices": indices, "material": 0, "mode": TRIANGLES,
                                       "targets": targets}]}]
    times = b.accessor((np.arange(n_frames, dtype=np.float64) / fps).astype(np.float32).reshape(-1, 1), F32, "SCALAR",
                       min_max=True)
    gltf["animations"] = [{"name": "Animation",
                           "channels": [{"sampler": 0, "target": {"node": 0, "path": "weights"}}],
                           "samplers": [{"input": times, "output": b.accessor(weights.reshape(-1, 1), F32, "SCALAR"),
                                         "interpolation": "LINEAR"}]}]
    b.write(path, gltf)


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
