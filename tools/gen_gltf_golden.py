"""Write tests/golden/panda_blender_small.glb: a small GLB in the exact layout of a file written by Blender's glTF exporter.

    python tools/gen_gltf_golden.py <actionmesh checkout>/assets/examples/panda/panda.glb

The source is the reference's example mesh (Khronos glTF Blender I/O; 9 606 vertices, a 1 MB JPEG texture), too large to
keep in the repository.  The fixture keeps its JSON as Blender wrote it (asset, scene, node, material, sampler, texture,
image entry, accessor types and component types, one bufferView per attribute) and changes only the data: the faces whose
corners all lie among the first KEEP_VERTICES vertices, the vertices they use (in their original order, with their
normals and UVs), and the texture re-encoded as a 64 x 64 JPEG.  Counts, offsets, lengths and POSITION min/max are
recomputed for the new data.
"""
from __future__ import annotations

import io
import json
import struct
import sys
from pathlib import Path

import numpy as np
from PIL import Image

ROOT = Path(__file__).resolve().parents[1]
OUT = ROOT / "tests" / "golden" / "panda_blender_small.glb"
KEEP_VERTICES = 1200
DTYPES = {5121: "<u1", 5123: "<u2", 5125: "<u4", 5126: "<f4"}
NCOMP = {"SCALAR": 1, "VEC2": 2, "VEC3": 3}


def main(src: str) -> None:
    data = Path(src).read_bytes()
    (jlen,) = struct.unpack_from("<I", data, 12)
    gltf = json.loads(data[20:20 + jlen])
    binary = data[20 + jlen + 8:]
    views = gltf["bufferViews"]

    def view(i):
        v = views[i]
        return binary[v.get("byteOffset", 0):v.get("byteOffset", 0) + v["byteLength"]]

    def accessor(i):
        a = gltf["accessors"][i]
        assert "byteStride" not in views[a["bufferView"]]
        return np.frombuffer(view(a["bufferView"]), DTYPES[a["componentType"]], a["count"] * NCOMP[a["type"]],
                             a.get("byteOffset", 0)).reshape(a["count"], -1)

    (prim,) = [p for m in gltf["meshes"] for p in m["primitives"]]
    faces = accessor(prim["indices"]).reshape(-1, 3).astype(np.int64)
    faces = faces[(faces < KEEP_VERTICES).all(1)]
    used = np.unique(faces)
    new_data = {prim["indices"]: np.searchsorted(used, faces).reshape(-1, 1)}
    for acc in prim["attributes"].values():
        new_data[acc] = accessor(acc)[used]
    (image,) = gltf["images"]
    jpeg = io.BytesIO()
    Image.open(io.BytesIO(view(image["bufferView"]))).convert("RGB").resize((64, 64), Image.LANCZOS).save(
        jpeg, format="JPEG", quality=90)

    out, blobs = bytearray(), {}
    for i, acc in enumerate(gltf["accessors"]):
        arr = np.ascontiguousarray(new_data[i], DTYPES[acc["componentType"]])
        acc["count"] = int(arr.shape[0])
        if "min" in acc:
            acc["min"], acc["max"] = arr.min(0).tolist(), arr.max(0).tolist()
        blobs[acc["bufferView"]] = arr.tobytes()
    blobs[image["bufferView"]] = jpeg.getvalue()
    for i, v in enumerate(views):
        out += b"\0" * (-len(out) % 4)
        v["byteOffset"], v["byteLength"] = len(out), len(blobs[i])
        out += blobs[i]
    out += b"\0" * (-len(out) % 4)
    gltf["buffers"] = [{"byteLength": len(out)}]
    js = json.dumps(gltf, separators=(",", ":")).encode()
    js += b" " * (-len(js) % 4)
    body = struct.pack("<II", len(js), 0x4E4F534A) + js + struct.pack("<II", len(out), 0x004E4942) + bytes(out)
    OUT.write_bytes(b"glTF" + struct.pack("<II", 2, 12 + len(body)) + body)
    print(f"{OUT}: {len(used)} vertices, {len(faces)} faces, {12 + len(body)} bytes")


if __name__ == "__main__":
    main(sys.argv[1])
