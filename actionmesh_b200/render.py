"""B200MeshVisualizer: the reference's ActionMeshVisualizer (actionmesh/render/visualizer.py) with the rendering on the GPU
(csrc/render.cu) instead of PyTorch3D.

`render(meshes, device, output_dir, input_frames)` writes `output_dir/grid_normal.mp4`: one grid frame per mesh, with a column
for the input frame (when given) and one per camera, each cell `image_size` square.  A camera cell is the mesh's interpolated
vertex normals seen from that camera, rasterized at 2x2 samples per pixel, composited on white with the 2x2 coverage as alpha,
exactly as the reference's Renderer + soft_normal_shading + make_normal_image produce it.  DESIGN.md §16 states every formula.

`render(..., modalities=("normal", "texture"), visual=...)` also writes `grid_texture.mp4`: the same rasterization shaded with
the glTF base colour (its texture, mip-mapped and filtered as the sampler says, or its factor) under a two-sided headlight,
each pixel the mean of its four samples (DESIGN.md §16, "Texture shading").  Each mesh is rasterized once per frame for
every modality.
Differences from the reference:
  - the video is encoded by OpenCV's `mp4v` writer (the reference uses imageio, which this project does not depend on): same
    file name, frame rate, frame size and frame count, different codec;
  - the reference's ambient "blue" image is never used by the visualizer and is not rendered, so `bg_color` (which only colours
    that image) is accepted and unused;
  - faces that repeat a corner are dropped before upload; they have zero area, so no pixel changes.
"""
from __future__ import annotations

import io
import logging
import math
from dataclasses import dataclass
from pathlib import Path
from typing import Optional

import numpy as np
import torch

from . import ops

logger = logging.getLogger(__name__)

ELEVATION_CYCLE = (70, 55, 85, 40)
FPS = 12
MODALITIES = ("normal", "texture")
MAX_TEXTURE_SIDE = 16384


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
    verts, faces, keep = _mesh_arrays(mesh)
    return verts, faces[keep].astype(np.int32)


def _mesh_arrays(mesh) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """`mesh_arrays` before the drop: (vertices, every face (F, 3) int64, the faces kept (F,) bool)."""
    with np.errstate(over="ignore"):
        verts = np.asarray(mesh.vertices, dtype=np.float64).reshape(-1, 3).astype(np.float32)
    faces = np.asarray(mesh.faces, dtype=np.int64).reshape(-1, 3)
    if not np.isfinite(verts).all():
        raise ValueError("render: the mesh has non-finite vertices (in float32)")
    if len(faces) and (faces.min() < 0 or faces.max() >= len(verts)):
        raise ValueError(f"render: face indices must lie in [0, {len(verts)})")
    keep = (faces[:, 0] != faces[:, 1]) & (faces[:, 1] != faces[:, 2]) & (faces[:, 0] != faces[:, 2])
    return verts, faces, keep


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


@dataclass
class TextureShading:
    """What the texture modality samples: the decoded base-colour image ((h, w, 3) uint8, or None for a flat colour), the
    sampler's glTF enums and the base colour factor (RGB)."""
    image: Optional[np.ndarray]
    mag_filter: int
    min_filter: int
    wrap_s: int
    wrap_t: int
    base_color: tuple


@dataclass
class MaterialShading:
    """What the texture modality samples for a `gltf.GltfMultiVisual`: one shading record per distinct (material, has UVs)
    pair that a primitive has, each a `TextureShading` whose `image` is an index into `images` (or None for a flat colour),
    the decoded images ((h, w, 3) uint8, each distinct image once) and the (F,) int32 record of every face."""
    records: list
    images: list
    face_record: np.ndarray


_DEFAULT_SAMPLER = (ops.LINEAR, ops.LINEAR_MIPMAP_NEAREST, ops.REPEAT, ops.REPEAT)


def _record(material: Optional[dict], textures: list, samplers: list, has_uv: bool, what: str, warned: Optional[set] = None):
    """(image source index or None, sampler enums, base colour) of one material as the texture modality uses it; an
    unusable texture is ignored with one warning (once per `what` when `warned` collects them)."""
    from .gltf import DEFAULT_MATERIAL

    if material is None:
        return None, _DEFAULT_SAMPLER, tuple(DEFAULT_MATERIAL["pbrMetallicRoughness"]["baseColorFactor"][:3])
    pbr = material.get("pbrMetallicRoughness", {})
    base = tuple(float(x) for x in pbr.get("baseColorFactor", [1.0, 1.0, 1.0, 1.0])[:3])
    info = pbr.get("baseColorTexture")
    if info is None:
        return None, _DEFAULT_SAMPLER, base
    tex = textures[info["index"]] if 0 <= info.get("index", -1) < len(textures) else {}
    why = ("it uses texCoord %s" % info["texCoord"] if info.get("texCoord", 0) != 0 else
           "its textureInfo has extensions (%s)" % ", ".join(info["extensions"]) if info.get("extensions") else
           "it has no image source" if "source" not in tex else
           "the mesh has no UVs" if not has_uv else None)
    if why is not None:
        if warned is None or what not in warned:
            logger.warning(f"render: {what} is ignored because {why}; shading with the base colour factor")
            if warned is not None:
                warned.add(what)
        return None, _DEFAULT_SAMPLER, base
    smp = samplers[tex["sampler"]] if "sampler" in tex else {}
    mode = (smp.get("magFilter", _DEFAULT_SAMPLER[0]), smp.get("minFilter", _DEFAULT_SAMPLER[1]),
            smp.get("wrapS", _DEFAULT_SAMPLER[2]), smp.get("wrapT", _DEFAULT_SAMPLER[3]))
    for value, allowed, name in zip(mode, (ops.MAG_FILTERS, ops.MIN_FILTERS, ops.WRAP_MODES, ops.WRAP_MODES),
                                    ("magFilter", "minFilter", "wrapS", "wrapT")):
        if value not in allowed:
            raise ValueError(f"render: sampler {name} {value} is not a glTF value ({', '.join(map(str, allowed))})")
    return tex["source"], mode, base


def _decode(data: bytes) -> np.ndarray:
    from PIL import Image

    with Image.open(io.BytesIO(data)) as img:
        if max(img.size) > MAX_TEXTURE_SIDE:
            raise ValueError(f"render: texture of {img.size[0]} x {img.size[1]} texels; each side must be <= {MAX_TEXTURE_SIDE}")
        return np.array(img.convert("RGB"))


def texture_shading(visual):
    """The base colour of a `gltf.GltfVisual` (or None) as the texture modality uses it -> a `TextureShading`; of a
    `gltf.GltfMultiVisual` -> a `MaterialShading`.

    No visual or no material: the animated GLB's default material colour.  A material: its `baseColorFactor` RGB, times
    its `baseColorTexture` when that is usable (no `texCoord` other than 0, no textureInfo `extensions`, an image source
    and UVs); an unusable texture is ignored with one warning (per material for a multi-primitive visual).  Images are
    decoded by Pillow to RGB (alpha ignored), each once.  Raises ValueError on an image side above 16384 or a sampler enum
    glTF does not define."""
    from .gltf import GltfMultiVisual, GltfVisual

    if isinstance(visual, GltfMultiVisual):
        return _material_shading(visual)
    if visual is not None and not isinstance(visual, GltfVisual):
        raise ValueError(f"render: visual must be a gltf.GltfVisual or gltf.GltfMultiVisual, got {type(visual).__name__}")
    visual = GltfVisual() if visual is None else visual
    source, mode, base = _record(visual.material, visual.textures, visual.samplers, visual.uv is not None,
                                 "the base colour texture")
    return TextureShading(None if source is None else _decode(visual.image_bytes[source]), *mode, base)


def _material_shading(visual) -> MaterialShading:
    """`texture_shading` of a `gltf.GltfMultiVisual`: records keyed by (material, has UVs) in first-use order."""
    keys, records, images, image_of, warned = {}, [], [], {}, set()
    prim_record = []
    for m, has_uv in zip(visual.primitive_material, np.asarray(visual.has_uv, bool)):
        key = (m, bool(has_uv))
        if key not in keys:
            material = None if m is None else visual.materials[m]
            source, mode, base = _record(material, visual.textures, visual.samplers, key[1],
                                         f"material {m}'s base colour texture", warned)
            if source is not None and source not in image_of:
                image_of[source] = len(images)
                images.append(_decode(visual.image_bytes[source]))
            keys[key] = len(records)
            records.append(TextureShading(None if source is None else image_of[source], *mode, base))
        prim_record.append(keys[key])
    counts = np.asarray(visual.face_ranges, np.int64).reshape(-1, 2)[:, 1]
    return MaterialShading(records, images, np.repeat(np.asarray(prim_record, np.int32), counts))


def _modalities(modalities) -> tuple:
    mods = tuple(modalities) if not isinstance(modalities, str) else (modalities,)
    unknown = [m for m in mods if m not in MODALITIES]
    if unknown or not mods or len(set(mods)) != len(mods):
        raise ValueError(f"render: modalities must be distinct names from {MODALITIES}, got {modalities!r}")
    return mods


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
    def render_frames(self, meshes: list, input_frames: Optional[list] = None, *, modalities=("normal",), visual=None):
        """The video's frames before encoding, per modality: host uint8 (n_frames, S, n_cols * S, 3), n_cols = cameras (+ 1
        for the input frame column when `input_frames` is given).  One modality -> its grid; several -> a tuple of grids in
        the order given.  `visual` (a `gltf.GltfVisual`, its uv one row per mesh vertex) gives "texture" its base colour; a
        `gltf.GltfMultiVisual`, whose ranges must fit every mesh, gives each face its primitive's material."""
        from .gltf import GltfMultiVisual, check_multi_visual

        mods = _modalities(modalities)
        S, n = self.image_size, len(meshes)
        full = [_mesh_arrays(m) for m in meshes]
        arrays = [(verts, faces[keep].astype(np.int32)) for verts, faces, keep in full]
        if isinstance(visual, GltfMultiVisual):
            for verts, faces, _ in full:
                try:
                    check_multi_visual(visual, len(verts), faces)
                except ValueError as exc:
                    raise ValueError(f"render: {exc}") from None
        uv = None if visual is None or getattr(visual, "uv", None) is None else np.asarray(visual.uv, dtype=np.float32)
        if uv is not None:
            if not np.isfinite(uv).all():
                raise ValueError("render: visual.uv has non-finite values")
            for verts, _ in arrays:
                if uv.shape != (len(verts), 2):
                    raise ValueError(f"render: visual.uv has shape {uv.shape}, but a mesh has {len(verts)} vertices")
        if self.device.type != "cuda":
            raise ops._lib.AmbError("B200MeshVisualizer renders on CUDA (sm_90a) only; there is no CPU fallback")
        if not self.cameras:
            raise ValueError("render: no camera selected")
        shading = texture_shading(visual) if "texture" in mods else None
        frames = resample_list(list(input_frames), n) if input_frames is not None else None
        col0 = 1 if frames is not None else 0
        n_cols = col0 + len(self.cameras)
        with torch.cuda.device(self.device):
            cams, focal = self._camera_table()
            grids = [torch.empty(n, S, n_cols * S, 3, dtype=torch.uint8, device=self.device) for _ in mods]
            tex, face_record = {}, None
            if isinstance(shading, MaterialShading):
                tex = self._material_tables(shading, uv)
            elif shading is not None:
                tex = dict(mag_filter=shading.mag_filter, min_filter=shading.min_filter, wrap_s=shading.wrap_s,
                           wrap_t=shading.wrap_t, base_color=shading.base_color)
                if shading.image is not None:  # the mip chain is built once per call
                    levels, table = ops.texture_levels(torch.from_numpy(shading.image).to(self.device))
                    tex.update(uv=torch.from_numpy(uv).to(self.device), levels=levels, table=table)
            for k, (verts, faces) in enumerate(arrays):
                v, f = torch.from_numpy(verts).to(self.device), torch.from_numpy(faces).to(self.device)  # no faces: white cells
                normals = ops.vertex_normals(v, f)
                pix_to_face = ops.rasterize(v, f, cams, focal, S)
                for grid, mod in zip(grids, mods):
                    if mod == "normal":
                        ops.shade_normals(v, f, normals, cams, focal, pix_to_face, out=grid[k], column=col0)
                    elif isinstance(shading, MaterialShading):
                        kept = shading.face_record[full[k][2]]
                        if face_record is None or not np.array_equal(kept, face_record[0]):  # meshes usually share faces
                            face_record = (kept, ops.face_records(kept, len(shading.records), self.device))
                        ops.shade_materials(v, f, normals, cams, focal, pix_to_face, face_record[1], out=grid[k],
                                            column=col0, **tex)
                    else:
                        ops.shade_texture(v, f, normals, cams, focal, pix_to_face, out=grid[k], column=col0, **tex)
            grids = [g.cpu() for g in grids]
        if frames is not None:
            for k, frame in enumerate(frames):
                cell = torch.from_numpy(_frame_rgb(frame, S))
                for grid in grids:
                    grid[k, :, :S] = cell
        return grids[0] if len(grids) == 1 else tuple(grids)

    def _material_tables(self, shading: MaterialShading, uv: Optional[np.ndarray]) -> dict:
        """`shade_materials`' records, levels and uv on the device: every distinct image's mip chain built once, all of
        them packed into one level buffer."""
        sizes = [ops.texture_chain_bytes(img.shape[1], img.shape[0]) for img in shading.images]
        levels = torch.empty(max(sum(sizes), 1), dtype=torch.uint8, device=self.device) if sizes else None
        tables, off = [], 0
        for img, size in zip(shading.images, sizes):
            tables.append(ops.texture_levels(torch.from_numpy(img).to(self.device), out=levels, offset=off)[1])
            off += size
        rows = [(None if r.image is None else tables[r.image], r.mag_filter, r.min_filter, r.wrap_s, r.wrap_t, r.base_color)
                for r in shading.records]
        textured = any(r.image is not None for r in shading.records)
        return dict(records=ops.shade_records(rows, levels, self.device), levels=levels,
                    uv=torch.from_numpy(uv).to(self.device) if textured else None)

    @torch.no_grad()
    def render(self, meshes: list, device=None, output_dir: str = ".", input_frames: Optional[list] = None, *,
               modalities=("normal",), visual=None) -> list[Path]:
        """Render the meshes and write output_dir/grid_{modality}.mp4 (12 fps) for each modality, in the order given ->
        their paths ([] when there are no meshes).  `device`, when given, replaces the constructor's; `visual` as for
        `render_frames`."""
        mods = _modalities(modalities)
        if device is not None:
            self.device = torch.device(device)
        if not len(meshes):
            return []
        grids = self.render_frames(meshes, input_frames, modalities=mods, visual=visual)
        grids = (grids,) if len(mods) == 1 else grids
        out_dir = Path(output_dir)
        out_dir.mkdir(parents=True, exist_ok=True)
        paths = []
        for mod, grid in zip(mods, grids):
            path = out_dir / f"grid_{mod}.mp4"
            write_video(grid.numpy(), path)
            logger.info(f"Saved render: {path}")
            paths.append(path)
        return paths
