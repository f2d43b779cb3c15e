"""Time B200MeshVisualizer.render_frames (mesh upload, vertex normals, rasterization of 3 views at 2S x 2S samples, shading,
grid download) with CUDA events, on a depth-9 Stage 0 mesh (~1.75 M faces, the rippled ball the geometry tests refine) and
on that mesh decimated to 40 000 faces, at 16 and 31 frames x 3 cameras x S = 256.  Then the texture modality on the
decimated mesh: normal only against normal + texture (a --texture-size square JPEG, decoded and mip-mapped in every call,
on spherical UVs), the two alternated.  Then per-face materials: the decimated mesh split into 8 primitives with 8
distinct --texture-size JPEGs against the same split mesh with one texture, normal + texture, the two alternated.  Prints
the card and its power limit with the numbers.

    python tools/render_probe.py [--repeats 3] [--texture-size 2048] [--materials-only]
"""
import io
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


class _Mesh:
    def __init__(self, vertices, faces):
        self.vertices, self.faces = vertices, faces


def _frames(base: np.ndarray, faces: np.ndarray, n: int) -> list:
    out = []
    for k in range(n):  # a twist about +Y growing with k, and a bob
        a = 0.03 * k * base[:, 1]
        x, z = base[:, 0] * np.cos(a) - base[:, 2] * np.sin(a), base[:, 0] * np.sin(a) + base[:, 2] * np.cos(a)
        out.append(_Mesh(np.stack([x, base[:, 1] + 0.01 * k, z], 1).astype(np.float32), faces))
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--image-size", type=int, default=256)
    ap.add_argument("--texture-size", type=int, default=2048)
    ap.add_argument("--materials-only", action="store_true", help="Only the per-face material comparison.")
    args = ap.parse_args()

    import geometry_exact as gx
    import triposg_vae_ref as ref
    from actionmesh_b200 import ops
    from actionmesh_b200.mesh_process import B200MeshPostprocessor
    from actionmesh_b200.render import B200MeshVisualizer
    from actionmesh_b200.triposg_vae import refine_octree

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"card: {q.stdout.strip() or torch.cuda.get_device_name()}")
    grid = refine_octree(gx.rippled_field, ref.BOUNDS, 9)
    gv, gf = ops.dual_marching_cubes(grid)
    del grid
    base = gv.cpu().numpy().astype(np.float64) * (2.01 / 504) - 1.005
    faces = gf.cpu().numpy().astype(np.int64)
    small = B200MeshPostprocessor(face_decimation=40_000, verbose=False).process_mesh(_Mesh(base, faces))
    meshes = {"depth-9": (base, faces), "decimated": (np.asarray(small.vertices), np.asarray(small.faces))}
    vis = B200MeshVisualizer(image_size=args.image_size)
    for name, (v, f) in meshes.items():
        for n in (16, 31) if not args.materials_only else ():
            clip = _frames(v, f, n)
            vis.render_frames(clip[:2])  # warm-up
            times = []
            for _ in range(args.repeats):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
                vis.render_frames(clip)
                e1.record()
                torch.cuda.synchronize()
                times.append(e0.elapsed_time(e1))
            ms = float(np.median(times))
            print(f"{name}: {len(f):,} faces, {n} frames x 3 views, S = {args.image_size}: {ms:.1f} ms per clip "
                  f"(min {min(times):.1f}), {ms / (3 * n):.2f} ms per view")

    v, f = meshes["decimated"]
    visual = _textured(v, args.texture_size)
    for n in (16, 31) if not args.materials_only else ():
        clip = _frames(v, f, n)
        runs = {("normal",): [], ("normal", "texture"): []}
        for mods in runs:
            vis.render_frames(clip[:2], modalities=mods, visual=visual)  # warm-up
        for _ in range(args.repeats):
            for mods, times in runs.items():
                times.append(_timed(lambda: vis.render_frames(clip, modalities=mods, visual=visual)))
        for mods, times in runs.items():
            ms = float(np.median(times))
            print(f"decimated: {len(f):,} faces, {n} frames x 3 views, S = {args.image_size}, {' + '.join(mods)}"
                  f"{f', {args.texture_size}^2 texture' if 'texture' in mods else ''}: {ms:.1f} ms per clip "
                  f"(min {min(times):.1f}, max {max(times):.1f})")


    from test_multi_material_cpu import split

    groups = np.array_split(np.arange(len(f)), 8)
    sv, sf, suv, vr, fr = split(v, f, _textured(v, 1).uv, groups)
    one, eight = _textured(sv, args.texture_size), _materials(sv, suv, vr, fr, args.texture_size)
    for n in (16, 31):
        clip = _frames(sv, sf, n)
        runs = {"1 texture": (one, []), "8 primitives, 8 textures": (eight, [])}
        for visual, _ in runs.values():
            vis.render_frames(clip[:2], modalities=("normal", "texture"), visual=visual)  # warm-up
        for _ in range(args.repeats):
            for visual, times in runs.values():
                times.append(_timed(lambda: vis.render_frames(clip, modalities=("normal", "texture"), visual=visual)))
        for name, (_, times) in runs.items():
            ms = float(np.median(times))
            print(f"split decimated: {len(sf):,} faces, {n} frames x 3 views, S = {args.image_size}, normal + texture, "
                  f"{name} of {args.texture_size}^2: {ms:.1f} ms per clip (min {min(times):.1f}, max {max(times):.1f})")


def _materials(v, uv, vertex_ranges, face_ranges, size: int):
    """A GltfMultiVisual: primitive p has material p with its own size x size JPEG (seeded per primitive)."""
    from actionmesh_b200.gltf import GltfMultiVisual

    P = len(vertex_ranges)
    jpegs = [_jpeg(size, seed) for seed in range(1, P + 1)]
    return GltfMultiVisual(vertex_ranges=vertex_ranges, face_ranges=face_ranges, uv=uv, has_uv=np.ones(P, bool),
                           primitive_material=list(range(P)),
                           materials=[{"pbrMetallicRoughness": {"baseColorTexture": {"index": p}}} for p in range(P)],
                           textures=[{"source": p} for p in range(P)], images=[{"mimeType": "image/jpeg"}] * P,
                           image_bytes=jpegs)


def _timed(fn) -> float:
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def _textured(v: np.ndarray, size: int):
    """A GltfVisual on spherical UVs with a size x size JPEG: a colour gradient with seeded noise."""
    from actionmesh_b200.gltf import GltfVisual

    c = v - v.mean(0)
    uv = np.stack([np.arctan2(c[:, 2], c[:, 0]) / (2 * np.pi) + 0.5,
                   np.arccos(np.clip(c[:, 1] / np.linalg.norm(c, axis=1), -1, 1)) / np.pi], 1).astype(np.float32)
    return GltfVisual(uv=uv, material={"pbrMetallicRoughness": {"baseColorTexture": {"index": 0}}},
                      textures=[{"source": 0}], images=[{"mimeType": "image/jpeg"}], image_bytes=[_jpeg(size, 0)])


def _jpeg(size: int, seed: int) -> bytes:
    """A size x size JPEG: a colour gradient with seeded noise."""
    from PIL import Image

    y, x = np.mgrid[0:size, 0:size]
    noise = np.random.default_rng(seed).integers(0, 48, (size, size, 3))
    img = np.stack([x * 200 // size, y * 200 // size, (x + y) * 100 // size], -1) + noise
    buf = io.BytesIO()
    Image.fromarray(img.astype(np.uint8)).save(buf, format="JPEG", quality=90)
    return buf.getvalue()


if __name__ == "__main__":
    main()
