"""A GLB reader for the tests, written from the glTF 2.0 specification and independent of `actionmesh_b200.gltf`.

`check_glb(path)` parses a file and asserts the structural rules a valid GLB meets (there is no glTF validator here):
header, chunk padding, buffer length, bufferView and accessor bounds and alignment, POSITION min/max, index range, morph
targets against mesh weights, and animation sampler inputs and outputs.  `read_animated(path)` reads back what
`write_animated_glb` writes.
"""
from __future__ import annotations

import json
import struct

import numpy as np

DTYPES = {5120: "<i1", 5121: "<u1", 5122: "<i2", 5123: "<u2", 5125: "<u4", 5126: "<f4"}
NCOMP = {"SCALAR": 1, "VEC2": 2, "VEC3": 3, "VEC4": 4}


def accessor(gltf: dict, binary: bytes, i: int) -> np.ndarray:
    """(count, n) array of accessor `i`, buffer 0 being the BIN chunk."""
    acc = gltf["accessors"][i]
    view = gltf["bufferViews"][acc["bufferView"]]
    dt, n = np.dtype(DTYPES[acc["componentType"]]), NCOMP[acc["type"]]
    stride = view.get("byteStride", n * dt.itemsize)
    start = view.get("byteOffset", 0) + acc.get("byteOffset", 0)
    rows = [np.frombuffer(binary, dt, n, start + k * stride) for k in range(acc["count"])] if stride != n * dt.itemsize \
        else [np.frombuffer(binary, dt, n * acc["count"], start)]
    return np.concatenate(rows).reshape(acc["count"], n) if rows else np.zeros((0, n), dt)


def check_glb(path) -> tuple[dict, bytes]:
    """Assert the structural rules on the GLB at `path` -> (JSON, BIN payload or b"")."""
    data = open(path, "rb").read()
    magic, version, length = struct.unpack_from("<4sII", data, 0)
    assert magic == b"glTF" and version == 2 and length == len(data)
    jlen, jtype = struct.unpack_from("<II", data, 12)
    assert jtype == 0x4E4F534A and jlen % 4 == 0
    raw = data[20:20 + jlen]
    text = raw.rstrip(b" ")
    assert raw[len(text):] == b" " * (jlen - len(text))           # padded with spaces
    gltf = json.loads(text)
    binary = b""
    off = 20 + jlen
    if off < length:
        blen, btype = struct.unpack_from("<II", data, off)
        assert btype == 0x004E4942 and blen % 4 == 0 and off + 8 + blen == length
        binary = data[off + 8:off + 8 + blen]
    buffers = gltf.get("buffers", [])
    if binary:
        assert buffers[0]["byteLength"] == len(binary) and "uri" not in buffers[0]
    else:
        assert not buffers
    used = 0
    for v in gltf.get("bufferViews", []):
        start = v.get("byteOffset", 0)
        assert v["buffer"] == 0 and start % 4 == 0 and start + v["byteLength"] <= len(binary)
        used = max(used, start + v["byteLength"])
    assert binary[used:] == b"\0" * (len(binary) - used)            # padded with zeros
    for a in gltf.get("accessors", []):
        view = gltf["bufferViews"][a["bufferView"]]
        item = np.dtype(DTYPES[a["componentType"]]).itemsize
        elem = NCOMP[a["type"]] * item
        stride = view.get("byteStride", elem)
        start = a.get("byteOffset", 0)
        assert start % item == 0 and a["count"] >= 1
        assert start + (a["count"] - 1) * stride + elem <= view["byteLength"]
    for mesh in gltf.get("meshes", []):
        for prim in mesh["primitives"]:
            pos = accessor(gltf, binary, prim["attributes"]["POSITION"])
            for acc_i in [prim["attributes"]["POSITION"]] + [t["POSITION"] for t in prim.get("targets", [])]:
                acc, x = gltf["accessors"][acc_i], accessor(gltf, binary, acc_i)
                assert acc["min"] == x.min(0).tolist() and acc["max"] == x.max(0).tolist()
                assert len(x) == len(pos)
            if "indices" in prim:
                assert accessor(gltf, binary, prim["indices"]).max() < len(pos)
            if "targets" in prim:
                assert len(prim["targets"]) == len(mesh["weights"])
    for anim in gltf.get("animations", []):
        for ch in anim["channels"]:
            smp = anim["samplers"][ch["sampler"]]
            t = accessor(gltf, binary, smp["input"])[:, 0]
            assert np.all(np.diff(t) > 0)
            acc_in = gltf["accessors"][smp["input"]]
            assert acc_in["min"] == [float(t.min())] and acc_in["max"] == [float(t.max())]
            n_out = gltf["accessors"][smp["output"]]["count"]
            if ch["target"]["path"] == "weights":
                mesh = gltf["meshes"][gltf["nodes"][ch["target"]["node"]]["mesh"]]
                assert n_out == len(t) * len(mesh["weights"])
    return gltf, binary


def image_bytes(gltf: dict, binary: bytes) -> list:
    out = []
    for img in gltf.get("images", []):
        v = gltf["bufferViews"][img["bufferView"]]
        out.append(binary[v.get("byteOffset", 0):v.get("byteOffset", 0) + v["byteLength"]])
    return out


def read_animated(path) -> dict:
    """base (V, 3), deltas (T, V, 3), faces, times (T,), weights (T, T), target names, material, uv, image bytes."""
    gltf, binary = check_glb(path)
    mesh = gltf["meshes"][gltf["nodes"][0]["mesh"]]
    prim = mesh["primitives"][0]
    smp = gltf["animations"][0]["samplers"][0]
    times = accessor(gltf, binary, smp["input"])[:, 0]
    uv = prim["attributes"].get("TEXCOORD_0")
    return {"gltf": gltf, "base": accessor(gltf, binary, prim["attributes"]["POSITION"]),
            "deltas": np.stack([accessor(gltf, binary, t["POSITION"]) for t in prim["targets"]]),
            "faces": accessor(gltf, binary, prim["indices"]).reshape(-1, 3),
            "times": times, "weights": accessor(gltf, binary, smp["output"]).reshape(len(times), -1),
            "interpolation": smp["interpolation"], "channel": gltf["animations"][0]["channels"][0]["target"],
            "target_names": mesh["extras"]["targetNames"], "material": gltf["materials"][prim["material"]],
            "uv": None if uv is None else accessor(gltf, binary, uv), "image_bytes": image_bytes(gltf, binary)}


def blender_frame(v: np.ndarray) -> np.ndarray:
    """What frame k of the reference's animated GLB shows for mesh vertices `v`: save_deformation's (x, y, z) ->
    (-z, x, y), then the +Y-up glTF export's (bx, by, bz) -> (bx, bz, -by).  float64."""
    v = np.asarray(v, dtype=np.float64)
    b = np.stack([-v[..., 2], v[..., 0], v[..., 1]], -1)
    return np.stack([b[..., 0], b[..., 2], -b[..., 1]], -1)


def check_animated(path, vertices, faces, fps=8) -> dict:
    """Assert that the animated GLB at `path` shows `blender_frame(vertices[k])` at time k / fps -> its contents."""
    a = read_animated(path)
    n = len(vertices)
    want = blender_frame(vertices)
    tol = 2.0 ** -22 * np.abs(want).max()
    for k in range(n):
        got = a["base"].astype(np.float64) + a["deltas"][k].astype(np.float64)
        assert np.abs(got - want[k]).max() <= tol, k
    assert np.array_equal(a["faces"], np.asarray(faces))
    assert np.array_equal(a["times"], (np.arange(n) / fps).astype(np.float32))
    assert np.array_equal(a["weights"], np.eye(n, dtype=np.float32))
    assert a["interpolation"] == "LINEAR" and a["channel"] == {"node": 0, "path": "weights"}
    assert a["target_names"] == [f"Frame_{k}" for k in range(n)]
    return a
