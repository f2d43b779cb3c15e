"""Frames for the pipeline from a video file, a glob pattern or a directory: the reference's `load_frames`
(actionmesh/io/video_input.py:74-262) without natsort.

    load_frames("clip.mp4")            every decoded frame, BGR -> RGBA (OpenCV)
    load_frames("frames/*.png")        the matching images in natural order
    load_frames("frames/")             *_image.png + *_mask.png pairs, else *.png, *.jpg, *.jpeg or *.webp

`stride` keeps every n-th frame and is applied before `max_frames`; timesteps are 0, 1, 2, ... (float32).  The result is
the pipeline's `ActionMeshInput`, so fewer than 16 frames fails its check.
"""
from __future__ import annotations

import logging
import os
import re
from pathlib import Path
from typing import Optional

import torch
from PIL import Image

from .pipeline import ActionMeshInput

logger = logging.getLogger(__name__)

VIDEO_EXTENSIONS = (".mp4", ".avi", ".mov")
# Tried in this order (the reference iterates a set, so its order depends on the hash seed).
IMAGE_EXTENSIONS = (".png", ".jpg", ".jpeg", ".webp")


def natural_sorted(names) -> list:
    """Sort by the digit runs of each name as numbers and the rest as lower-case text (natsort's default order on these
    file names)."""
    def key(name):
        parts = re.split(r"(\d+)", os.path.basename(str(name)))
        return [(0, int(p), "") if p.isdigit() else (1, 0, p.lower()) for p in parts if p != ""]
    return sorted(names, key=key)


def _select(items: list, max_frames: Optional[int], stride: int) -> list:
    items = items[::stride]
    return items if max_frames is None else items[:max_frames]


def _input(frames: list) -> ActionMeshInput:
    return ActionMeshInput(frames=frames, timesteps=torch.arange(len(frames), dtype=torch.float32))


def load_from_image_mask_pairs(directory, max_frames: Optional[int] = None, stride: int = 1) -> ActionMeshInput:
    """xxx_image.png + xxx_mask.png pairs in `sorted` order; the mask (resized with LANCZOS to the image's size when they
    differ) becomes the image's alpha."""
    directory = Path(directory)
    image_files = sorted(directory.glob("*_image.png"))
    if not image_files:
        raise ValueError(f"No *_image.png files found in '{directory}'")
    frames = []
    for image_file in _select(image_files, max_frames, stride):
        mask_file = directory / f"{image_file.stem.replace('_image', '')}_mask.png"
        if not mask_file.exists():
            raise ValueError(f"No mask found for {image_file.name}: expected {mask_file}")
        image = Image.open(image_file).convert("RGB")
        mask = Image.open(mask_file).convert("L")
        if image.size != mask.size:
            mask = mask.resize(image.size, Image.LANCZOS)
        rgba = image.copy()
        rgba.putalpha(mask)
        frames.append(rgba)
    logger.info(f"Loaded {len(frames)} frames from image+mask pairs: {directory}")
    return _input(frames)


def load_from_image_dir(path_pattern, max_frames: Optional[int] = None, stride: int = 1) -> ActionMeshInput:
    """The images matching a glob pattern ("dir/*.png"), in natural order, as RGBA."""
    path_pattern = Path(path_pattern)
    image_paths = natural_sorted(path_pattern.parent.glob(path_pattern.name))
    if not image_paths:
        raise ValueError(f"No images found matching '{path_pattern}'")
    frames = [Image.open(p).convert("RGBA") for p in _select(image_paths, max_frames, stride)]
    logger.info(f"Loaded {len(frames)} frames from image folder: {path_pattern.parent}")
    return _input(frames)


def load_from_video(video_path, max_frames: Optional[int] = None, stride: int = 1) -> ActionMeshInput:
    """Every `stride`-th frame OpenCV decodes, BGR -> RGBA, up to `max_frames`."""
    import cv2

    video_path = Path(video_path)
    if not video_path.exists():
        raise FileNotFoundError(f"Video file not found: {video_path}")
    cap = cv2.VideoCapture(str(video_path))
    if not cap.isOpened():
        raise RuntimeError(f"Failed to open video: {video_path}")
    frames, frame_idx = [], 0
    try:
        while max_frames is None or len(frames) < max_frames:
            ret, frame = cap.read()
            if not ret:
                break
            if frame_idx % stride == 0:
                frames.append(Image.fromarray(cv2.cvtColor(frame, cv2.COLOR_BGR2RGBA)))
            frame_idx += 1
    finally:
        cap.release()
    if not frames:
        raise ValueError(f"No frames could be read from video: {video_path}")
    logger.info(f"Loaded {len(frames)} frames from video: {video_path}")
    return _input(frames)


def load_frames(path, max_frames: Optional[int] = None, stride: int = 1) -> ActionMeshInput:
    """A video file (.mp4, .avi, .mov), a glob pattern (contains * or ?) or a directory -> `ActionMeshInput`.

    FileNotFoundError: a missing video.  RuntimeError: a video OpenCV cannot open.  ValueError: no frames, or a path
    that is none of the three."""
    path = Path(path)
    if "*" in str(path) or "?" in str(path):
        return load_from_image_dir(path, max_frames=max_frames, stride=stride)
    if path.suffix.lower() in VIDEO_EXTENSIONS:
        return load_from_video(path, max_frames=max_frames, stride=stride)
    if path.is_dir():
        if any(path.glob("*_mask.png")):
            return load_from_image_mask_pairs(path, max_frames=max_frames, stride=stride)
        for ext in IMAGE_EXTENSIONS:
            if any(path.glob(f"*{ext}")):
                return load_from_image_dir(path / f"*{ext}", max_frames=max_frames, stride=stride)
        raise ValueError(f"No images found in directory: {path}")
    raise ValueError(f"Unsupported input: {path}. Expected video file, image pattern, or directory.")
