"""B200MeshVisualizer: the reference's ActionMeshVisualizer (actionmesh/render/visualizer.py) with the rendering on the GPU
(csrc/render.cu) instead of PyTorch3D.

`render(meshes, device, output_dir, input_frames)` writes `output_dir/grid_normal.mp4`: one grid frame per mesh, with a column
for the input frame (when given) and one per camera, each cell `image_size` square.  A camera cell is the mesh's interpolated
vertex normals seen from that camera, rasterized at 2x2 samples per pixel, composited on white with the 2x2 coverage as alpha,
exactly as the reference's Renderer + soft_normal_shading + make_normal_image produce it.  DESIGN.md §16 states every formula.
Differences from the reference:
  - the video is encoded by OpenCV's `mp4v` writer (the reference uses imageio, which this project does not depend on): same
    file name, frame rate, frame size and frame count, different codec;
  - the reference's ambient "blue" image is never used by the visualizer and is not rendered, so `bg_color` (which only colours
    that image) is accepted and unused;
  - faces that repeat a corner are dropped before upload; they have zero area, so no pixel changes.
"""
from __future__ import annotations

import logging
import math
from pathlib import Path
from typing import Optional

import numpy as np
import torch

from . import ops

logger = logging.getLogger(__name__)

ELEVATION_CYCLE = (70, 55, 85, 40)
FPS = 12


def uniform_cameras(distance: float = 3.0, n_cameras: int = 16,
                    focal_length: float = 2.1875) -> dict[str, tuple[np.ndarray, np.ndarray, float]]:
    """{"U000": (R (3, 3), T (3,), f), ...} float32, mirroring the reference's get_uniform_camera (render/cameras.py:114-139):
    camera i sits at elevation [70, 55, 85, 40][i % 4] degrees from +Y and azimuth i / n * 360 degrees, looks at the origin
    with +Y up; R has columns x, y, z of the look-at frame and T = -C R, so X_view = X R + T."""
    cams = {}
    for i in range(n_cameras):
        theta, phi = math.radians(i / n_cameras * 360), math.radians(ELEVATION_CYCLE[i % len(ELEVATION_CYCLE)])
        c = np.array([distance * math.sin(phi) * math.cos(theta), distance * math.cos(phi),
                      -distance * math.sin(phi) * math.sin(theta)], dtype=np.float32)
        z = -c / np.linalg.norm(c)
        x = np.cross(np.array([0, 1, 0], dtype=np.float32), z)
        x = x / np.linalg.norm(x)
        y = np.cross(z, x)
        y = y / np.linalg.norm(y)
        R = np.stack([x, y, z], axis=1).astype(np.float32)
        cams[f"U{i:03d}"] = (R, (-c @ R).astype(np.float32), float(focal_length))
    return cams


def resample_list(items: list, target_length: int) -> list:
    """The reference's nearest resampling of a list to `target_length` items (render/utils.py:16-36)."""
    if not items or target_length <= 0:
        return []
    if target_length == 1:
        return [items[0]]
    n_in = len(items)
    return [items[round(i * (n_in - 1) / (target_length - 1) + 1e-4)] for i in range(target_length)]


def mesh_arrays(mesh) -> tuple[np.ndarray, np.ndarray]:
    """(vertices (V, 3) float32, faces (F', 3) int32) of anything with .vertices / .faces, with the faces that repeat a corner
    dropped.  Raises ValueError on a face index outside [0, V) or a non-finite vertex."""
    with np.errstate(over="ignore"):
        verts = np.asarray(mesh.vertices, dtype=np.float64).reshape(-1, 3).astype(np.float32)
    faces = np.asarray(mesh.faces, dtype=np.int64).reshape(-1, 3)
    if not np.isfinite(verts).all():
        raise ValueError("render: the mesh has non-finite vertices (in float32)")
    if len(faces) and (faces.min() < 0 or faces.max() >= len(verts)):
        raise ValueError(f"render: face indices must lie in [0, {len(verts)})")
    keep = (faces[:, 0] != faces[:, 1]) & (faces[:, 1] != faces[:, 2]) & (faces[:, 0] != faces[:, 2])
    return verts, faces[keep].astype(np.int32)


def _frame_rgb(frame, size: int) -> np.ndarray:
    """An input frame as the reference's grid shows it: Pillow's default resize to size x size, RGB channels (alpha dropped
    without compositing)."""
    from PIL import Image

    img = frame if isinstance(frame, Image.Image) else Image.fromarray(np.asarray(frame))
    return np.array(img.resize((size, size)).convert("RGBA"))[..., :3]


def write_video(frames: np.ndarray, path: Path, fps: int = FPS) -> None:
    """(n, H, W, 3) uint8 RGB -> an mp4 (OpenCV, mp4v)."""
    import cv2

    n, h, w, _ = frames.shape
    writer = cv2.VideoWriter(str(path), cv2.VideoWriter_fourcc(*"mp4v"), fps, (w, h))
    if not writer.isOpened():
        raise RuntimeError(f"cannot open {path} for writing")
    try:
        for k in range(n):
            writer.write(np.ascontiguousarray(frames[k, :, :, ::-1]))
    finally:
        writer.release()


class B200MeshVisualizer:
    """Drop-in for the reference's `ActionMeshVisualizer` (same constructor and `render(meshes, device, output_dir,
    input_frames)`), rendering on `device`."""

    def __init__(self, image_size: int = 256, bg_color: tuple[float, float, float] = (1.0, 1.0, 1.0),
                 cameras: list[str] = ["U000", "U004", "U008"], *, device="cuda"):
        self.image_size = int(image_size)
        self.bg_color = tuple(bg_color)
        self.cameras = {k: v for k, v in uniform_cameras(distance=3.0).items() if k in cameras}
        self.device = torch.device(device)

    def _camera_table(self) -> tuple[torch.Tensor, float]:
        table = np.stack([np.concatenate([R.reshape(-1), T]) for R, T, _ in self.cameras.values()]).astype(np.float32)
        focal = {f for _, _, f in self.cameras.values()}
        assert len(focal) == 1, "cameras must share one focal length"
        return torch.from_numpy(table).to(self.device), focal.pop()

    @torch.no_grad()
    def render_frames(self, meshes: list, input_frames: Optional[list] = None) -> torch.Tensor:
        """The video's frames before encoding -> host uint8 (n_frames, S, n_cols * S, 3), n_cols = cameras (+ 1 for the input
        frame column when `input_frames` is given)."""
        if self.device.type != "cuda":
            raise ops._lib.AmbError("B200MeshVisualizer renders on CUDA (sm_90a) only; there is no CPU fallback")
        if not self.cameras:
            raise ValueError("render: no camera selected")
        S, n = self.image_size, len(meshes)
        arrays = [mesh_arrays(m) for m in meshes]
        frames = resample_list(list(input_frames), n) if input_frames is not None else None
        col0 = 1 if frames is not None else 0
        n_cols = col0 + len(self.cameras)
        with torch.cuda.device(self.device):
            cams, focal = self._camera_table()
            grid = torch.empty(n, S, n_cols * S, 3, dtype=torch.uint8, device=self.device)
            for k, (verts, faces) in enumerate(arrays):
                v, f = torch.from_numpy(verts).to(self.device), torch.from_numpy(faces).to(self.device)  # no faces: white cells
                normals = ops.vertex_normals(v, f)
                pix_to_face = ops.rasterize(v, f, cams, focal, S)
                ops.shade_normals(v, f, normals, cams, focal, pix_to_face, out=grid[k], column=col0)
            grid = grid.cpu()
        if frames is not None:
            for k, frame in enumerate(frames):
                grid[k, :, :S] = torch.from_numpy(_frame_rgb(frame, S))
        return grid

    @torch.no_grad()
    def render(self, meshes: list, device=None, output_dir: str = ".", input_frames: Optional[list] = None) -> list[Path]:
        """Render the meshes and write output_dir/grid_normal.mp4 (12 fps) -> [its path] ([] when there are no meshes).
        `device`, when given, replaces the constructor's."""
        if device is not None:
            self.device = torch.device(device)
        if not len(meshes):
            return []
        grid = self.render_frames(meshes, input_frames)
        out_dir = Path(output_dir)
        out_dir.mkdir(parents=True, exist_ok=True)
        path = out_dir / "grid_normal.mp4"
        write_video(grid.numpy(), path)
        logger.info(f"Saved render: {path}")
        return [path]
