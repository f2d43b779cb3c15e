"""Time B200MeshVisualizer.render_frames (mesh upload, vertex normals, rasterization of 3 views at 2S x 2S samples, shading,
grid download) with CUDA events, on a depth-9 Stage 0 mesh (~1.75 M faces, the rippled ball the geometry tests refine) and
on that mesh decimated to 40 000 faces, at 16 and 31 frames x 3 cameras x S = 256.  Prints the card and its power limit
with the numbers.

    python tools/render_probe.py [--repeats 3]
"""
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
        for n in (16, 31):
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


if __name__ == "__main__":
    main()
