"""ActionMeshB200Pipeline / Stage1Pipeline / AnimationPipeline — `ActionMeshPipeline.__call__` (reference
actionmesh/pipeline.py:602-685) on the CUDA path.  `Stage1Pipeline` is DinoV2 context for all frames (`encode_all_frames`,
:232-245), then the autoregressive Stage-I denoising over 16-frame windows (`generate_3d_latents` :435-508 ->
`_denoise_latents` :247-314), from the anchor latent in a seeded `LatentBank`, exactly the object `init_banks_from_anchor`
hands to `generate_3d_latents` in the reference (:661,:672).  `AnimationPipeline` adds Stage II (`generate_mesh_animation`
:510-600 -> `_decode_displacement` :316-385) on the CUDA autoencoder: the anchor mesh comes in as vertex features
(positions + unit normals, mesh_processor.py:85-101) and the result is a `VertexBank` (all output meshes share the anchor's
faces, so only vertices are produced).

`ActionMeshB200Pipeline` is seam 4 (SURVEY 8(b)): the reference's constructor and `__call__(input, seed, stage_0_steps,
face_decimation, floaters_threshold, stage_1_steps, guidance_scales, anchor_idx) -> list of meshes` (pipeline.py:47-53,
602-613) built from `actionmesh_b200*.yaml` through the same `_target_` plumbing.  `ActionMeshB200Pipeline.from_pretrained(
"pretrained_weights")` builds every stage from the reference's checkpoint directories: background removal
(background_removal.py), cropping (preprocess.py), Stage 0 (stage0.py, triposg_vae.py), mesh post-processing
(mesh_process.py), DinoV2, Stage I and Stage II.  The constructor instead takes the first three as injected components.
IO and rendering stay on the reference.
"""
from __future__ import annotations

import os
from dataclasses import dataclass
from typing import Callable, List, Optional

import numpy as np
import torch

from ._lib import AmbError
from .config import DEFAULT_CONFIG_DIR, get_target, instantiate, load_config
from .denoiser import B200Denoiser
from .guidance import ClassifierFreeGuidance
from .image_encoder import B200ImageEncoder
from .scheduler import B200SchedulerFlow
from .windows import (LatentBank, VertexBank, apply_scaling, chunk_from, get_scaling, interpolate_timesteps)


MIN_FRAMES = 16  # actionmesh/io/video_input.py:24


@dataclass
class ActionMeshInput:
    """Same fields and checks as the reference's `ActionMeshInput` (actionmesh/io/video_input.py:27-55): N >= 16 RGB(A) PIL
    frames and their float32 CPU timesteps.  The pipeline accepts the reference's own dataclass as well (duck-typed)."""
    frames: list
    timesteps: torch.Tensor

    def __post_init__(self) -> None:
        assert len(self.frames) >= MIN_FRAMES, f"At least {MIN_FRAMES} frames are required, got {len(self.frames)}"
        assert self.timesteps.ndim == 1, f"Expected 1D timesteps, got {self.timesteps.ndim}D"
        assert len(self.frames) == self.timesteps.shape[0], \
            f"Number of frames ({len(self.frames)}) must match timesteps ({self.timesteps.shape[0]})"
        assert self.timesteps.dtype == torch.float32, f"Expected float32 timesteps, got {self.timesteps.dtype}"
        assert self.timesteps.device.type == "cpu", f"Expected CPU timesteps, got {self.timesteps.device}"

    @property
    def n_frames(self) -> int:
        return len(self.frames)

    def get(self, indices: torch.Tensor) -> "VideoInput":
        return VideoInput([self.frames[int(i)] for i in indices], self.timesteps[indices])


@dataclass
class VideoInput:
    """The part of `ActionMeshInput` (actionmesh/io/video_input.py:27-55) Stage I consumes: frames + float timesteps."""
    frames: list
    timesteps: torch.Tensor  # (T,) fp32, CPU like the reference (video_input.py:53-55)

    @property
    def n_frames(self) -> int:
        return len(self.frames)

    def get(self, indices: torch.Tensor) -> "VideoInput":
        return VideoInput([self.frames[int(i)] for i in indices], self.timesteps[indices])


class Stage1Pipeline:
    def __init__(self, denoiser: B200Denoiser, scheduler: B200SchedulerFlow, cf_guidance: ClassifierFreeGuidance,
                 image_encoder: Optional[B200ImageEncoder] = None, temporal_context_size: int = 16,
                 sliding_window_denoiser: int = 15, anchor_idx: int = 0, latent_shape=(2048, 64)):
        self.temporal_3D_denoiser = denoiser
        self.scheduler = scheduler
        self.cf_guidance = cf_guidance
        self.image_encoder = image_encoder
        self.temporal_context_size = temporal_context_size
        self.sliding_window_denoiser = sliding_window_denoiser
        self.anchor_idx = anchor_idx
        self._denoiser_latent_shape = list(latent_shape)

    @property
    def device(self) -> torch.device:
        return self.temporal_3D_denoiser.device

    def encode_all_frames(self, input: VideoInput) -> torch.Tensor:
        """(T, S, D) context for all frames (pipeline.py:232-245)."""
        return self.image_encoder.encode_images(input.frames)

    def _denoise_latents(self, input: VideoInput, context: torch.Tensor, latent_bank: LatentBank, seed: int = 44,
                         step_callback: Optional[Callable[[int, int], None]] = None) -> torch.Tensor:
        """One AR window (pipeline.py:247-314)."""
        generator = torch.Generator(device=self.device).manual_seed(seed)
        cond_latents, cond_mask = latent_bank.get(timesteps=input.timesteps, device=self.device, add_batch_dim=True)
        init_noise = self.scheduler.get_noise(batch_size=1, latent_shape=self._denoiser_latent_shape,
                                              n_timesteps=input.n_frames, generator=generator, device=self.device)
        m = cond_mask[..., None, None].to(torch.float32)
        init_latent = cond_latents * m + init_noise * (1.0 - m)  # window set-up, once per window (pipeline.py:297)
        return self.scheduler.denoise(self.temporal_3D_denoiser, self.cf_guidance, init_latent=init_latent,
                                      context=context[None], mask=cond_mask.to(init_latent.dtype),
                                      framestep=input.timesteps[None], device=self.device, disable_prog=True,
                                      step_callback=step_callback)

    def generate_3d_latents(self, input: VideoInput, context: torch.Tensor, latent_bank: LatentBank, seed: int = 44,
                            step_callback: Optional[Callable[[int, int, int, int], None]] = None) -> LatentBank:
        """Serial AR windows, seed + i per window (pipeline.py:435-508)."""
        windows = chunk_from(start=self.anchor_idx, total=input.n_frames, size=self.temporal_context_size,
                             slide=self.sliding_window_denoiser)
        for i, idx in enumerate(windows):
            cb = None
            if step_callback is not None:
                cb = (lambda step, total, _i=i, _n=len(windows): step_callback(step, total, _i, _n))
            win = input.get(idx)
            lat = self._denoise_latents(win, context[idx.to(context.device)], latent_bank, seed=seed + i, step_callback=cb)
            latent_bank.update(latents=lat, timesteps=win.timesteps)
        return latent_bank

    @torch.no_grad()
    def __call__(self, input: VideoInput, anchor_latent: torch.Tensor, seed: int = 44,
                 stage_1_steps: Optional[int] = None, guidance_scales: Optional[List[float]] = None,
                 anchor_idx: Optional[int] = None, context: Optional[torch.Tensor] = None) -> LatentBank:
        """Stage-I part of ActionMeshPipeline.__call__ (pipeline.py:637-675): same override plumbing, returns the bank of
        denoised latents (what Stage II consumes)."""
        if stage_1_steps is not None:
            self.scheduler.num_inference_steps = stage_1_steps
        if guidance_scales is not None:
            self.cf_guidance.guidance_scales = guidance_scales
        if anchor_idx is not None:
            self.anchor_idx = anchor_idx
        bank = LatentBank(empty_dims=tuple(self._denoiser_latent_shape))
        bank.update(timesteps=input.timesteps[self.anchor_idx:self.anchor_idx + 1],
                    latents=anchor_latent.to(device=self.device, dtype=torch.float32))
        if context is None:
            context = self.encode_all_frames(input)
        return self.generate_3d_latents(input, context, bank, seed=seed)



class AnimationPipeline(Stage1Pipeline):
    """Stage I + Stage II of `ActionMeshPipeline.__call__` (pipeline.py:637-683) on the CUDA path."""

    def __init__(self, denoiser, scheduler, cf_guidance, autoencoder, image_encoder=None, *,
                 sliding_window_autoencoder: int = 15, subsampling_level: int = 1,
                 normals_fn: Optional[Callable[[torch.Tensor], torch.Tensor]] = None, **kwargs):
        super().__init__(denoiser, scheduler, cf_guidance, image_encoder, **kwargs)
        self.temporal_3D_vae = autoencoder
        self.sliding_window_autoencoder = sliding_window_autoencoder
        self.subsampling_level = subsampling_level
        # (V, 3) vertices -> (V, 3) unit vertex normals of the deformed anchor mesh; the reference gets them from
        # trimesh (`mesh.vertex_normals`, mesh_processor.py:98).  Needed only when a clip spans more than one AR window.
        self.normals_fn = normals_fn

    def _decode_displacement(self, latents: torch.Tensor, window_timesteps: torch.Tensor, source_alpha: torch.Tensor,
                             target_alphas: torch.Tensor, vertex_features: torch.Tensor,
                             step_callback: Optional[Callable[[int, int], None]] = None) -> torch.Tensor:
        """One AR window (pipeline.py:316-385): (V, 3|6) anchor features -> (T_out, V, 3) deformed vertices."""
        q = vertex_features[None].to(self.device)
        disp = self.temporal_3D_vae(latent=latents, framestep=window_timesteps, source_alpha=source_alpha,
                                    target_alphas=target_alphas, query=q, step_callback=step_callback)
        return self.temporal_3D_vae.apply_displacement(vertex=q[..., :3], displacement=disp)[0]

    def generate_mesh_animation(self, latent_bank: LatentBank, vertex_bank: VertexBank, anchor_normals: torch.Tensor,
                                step_callback: Optional[Callable[[int, int, int, int], None]] = None) -> VertexBank:
        """Serial AR windows over the denoised latents (pipeline.py:510-600).  `vertex_bank` holds the anchor vertices at
        the anchor timestep; `anchor_normals` are its unit vertex normals."""
        windows = chunk_from(start=self.anchor_idx, total=latent_bank.n_timesteps,
                             size=self.temporal_3D_vae.config.temporal_context_size, slide=self.sliding_window_autoencoder)
        all_ts = latent_bank.get_ordered_timesteps()
        anchor_t = sorted(vertex_bank.timesteps)[0] if vertex_bank.n_timesteps == 1 else None
        for wi, idx in enumerate(windows):
            wts = all_ts[idx][None]                                             # (1, T)
            lat, _ = latent_bank.get(timesteps=wts[0], device=self.device, add_batch_dim=True)
            verts = vertex_bank.get(timesteps=wts[:, 0])[0]
            assert verts is not None, "Anchor mesh should be in the vertex bank"
            if anchor_t is not None and abs(float(wts[0, 0]) - anchor_t) < 1e-5:
                normals = anchor_normals
            elif self.normals_fn is not None:
                normals = self.normals_fn(verts)
            else:
                raise ValueError("a clip spanning several AR windows needs `normals_fn` (vertex normals of the deformed anchor)")
            feats = torch.cat([verts.to(self.device, torch.float32), normals.to(self.device, torch.float32)], dim=-1)
            out_ts = interpolate_timesteps(wts, subsampling_level=self.subsampling_level, device="cpu", drop_first=True)
            t_min, t_range = get_scaling(wts)
            cb = None
            if step_callback is not None:
                cb = (lambda step, total, _i=wi, _n=len(windows): step_callback(step, total, _i, _n))
            v = self._decode_displacement(lat, wts, apply_scaling(wts[:, 0], t_min, t_range),
                                          apply_scaling(out_ts, t_min, t_range), feats, step_callback=cb)
            vertex_bank.update(timesteps=out_ts[0], vertices=list(v))
        return vertex_bank

    def __call__(self, input: VideoInput, anchor_latent: torch.Tensor, anchor_vertices: torch.Tensor,
                 anchor_normals: torch.Tensor, seed: int = 44, stage_1_steps: Optional[int] = None,
                 guidance_scales: Optional[List[float]] = None, anchor_idx: Optional[int] = None,
                 context: Optional[torch.Tensor] = None, faces=None):
        """-> (LatentBank, VertexBank): Stage I then Stage II for every output timestep."""
        bank = super().__call__(input, anchor_latent, seed=seed, stage_1_steps=stage_1_steps,
                                guidance_scales=guidance_scales, anchor_idx=anchor_idx, context=context)
        vb = VertexBank(faces=faces)
        vb.update(timesteps=input.timesteps[self.anchor_idx:self.anchor_idx + 1],
                  vertices=[anchor_vertices.to(self.device, torch.float32)])
        return bank, self.generate_mesh_animation(bank, vb, anchor_normals)


# ---------------------------------------------------------------------------------------------------- seam 4: the pipeline
class PassThroughMeshProcess:
    """Stand-in for the reference's CPU `MeshPostprocessor` (actionmesh/preprocessing/mesh_processor.py:374, decimation +
    floater removal — out of scope): same constructor arguments / mutable attributes, `process_mesh` returns its input."""

    def __init__(self, face_decimation: int = 40000, floaters_threshold: float = 0.02):
        self.face_decimation = face_decimation
        self.floaters_threshold = floaters_threshold

    def process_mesh(self, mesh, seed: int = 44):
        return mesh


@dataclass
class Mesh:
    """Minimal mesh record returned when `trimesh` is not installed: (V, 3) float32 vertices + (F, 3) int faces (numpy)."""
    vertices: "object"
    faces: "object"


def _vertex_normals(vertices: torch.Tensor, faces: torch.Tensor) -> torch.Tensor:
    """Unit vertex normals of a triangle mesh (area-weighted face normals).  Used for the deformed anchor of clips spanning
    several AR windows when trimesh is unavailable (the reference reads trimesh's `vertex_normals`, mesh_processor.py:98)."""
    v0, v1, v2 = (vertices[faces[:, i]] for i in range(3))
    fn = torch.cross(v1 - v0, v2 - v0, dim=-1)
    vn = torch.zeros_like(vertices)
    for i in range(3):
        vn.index_add_(0, faces[:, i], fn)
    return vn / vn.norm(dim=-1, keepdim=True).clamp_min(1e-12)


def vertex_normals(verts: torch.Tensor, faces: torch.Tensor) -> torch.Tensor:
    """(V, 3) fp32 unit vertex normals: trimesh's `vertex_normals`, the reference's source (mesh_processor.py:98), or
    `_vertex_normals` when trimesh is not installed."""
    try:
        import trimesh

        return torch.as_tensor(trimesh.Trimesh(vertices=verts.cpu().numpy(), faces=faces.cpu().numpy(),
                                               process=False).vertex_normals.copy(), dtype=torch.float32)
    except ImportError:
        return _vertex_normals(verts.to(torch.float32), faces.to(verts.device))


class ActionMeshB200Pipeline:
    """Drop-in for `ActionMeshPipeline` on the CUDA path: same constructor arguments, `.to(device)`, and `__call__`
    signature / return value (reference actionmesh/pipeline.py:47-53,205,602-685).

    Built from `actionmesh_b200.yaml` / `actionmesh_b200_fast.yaml` (the reference's YAML with the `_target_`s re-pointed):
    scheduler, guidance, mesh post-process are instantiated at construction like the reference (:98-110); denoiser, image
    encoder and autoencoder are resolved from their `_target_`s and loaded from `weights_dir` by `.to()` (or assigned
    directly — `pipe.temporal_3D_denoiser = model` — when weights do not come from disk).

    `from_pretrained(weights_root)` builds the whole pipeline from the reference's checkpoint layout.  The constructor
    takes these components as injected arguments instead (any object with the same surface):
      image_to_3d(image=, generator=, num_inference_steps=, guidance_scale=) -> (anchor_latent, anchor_mesh)   [TripoSGStage0]
      background_removal.process_images(frames), image_process.process_images(frames)                          [optional]
    `anchor_mesh` needs `.vertices`, `.faces` and `.vertex_normals` (the trimesh attributes the reference reads)."""

    def __init__(self, config_name: str = "actionmesh_b200.yaml", config_dir: Optional[str] = None,
                 dtype: torch.dtype = torch.bfloat16, lazy_loading: bool = False, *, image_to_3d=None,
                 background_removal=None, image_process=None, weights_dir: str = "pretrained_weights/ActionMesh",
                 config_updates: Optional[dict] = None):
        self.cfg = load_config(config_name, config_dir or DEFAULT_CONFIG_DIR, updates=config_updates)
        self._actionmesh_weights_dir = weights_dir
        self.image_to_3d_pipe = image_to_3d
        self.background_removal = background_removal
        self.image_process = image_process
        self.temporal_3D_denoiser = None
        self.image_encoder = None
        self.temporal_3D_vae = None
        self._denoiser_latent_shape = tuple(self.cfg.denoiser_latent_shape)
        self.mesh_process = instantiate(self.cfg.model.mesh_process, _convert_="partial")()
        self.scheduler = instantiate(self.cfg.model.scheduler, _convert_="partial")()
        self.cf_guidance = instantiate(self.cfg.model.cf_guidance, _convert_="partial")()
        self._target_device = torch.device("cpu")
        self._dtype = dtype            # accepted for signature compatibility: the CUDA path owns its precision recipe
        self._lazy_loading = lazy_loading
        self._loaders: dict = {}       # attribute -> callable building it from a checkpoint (set by from_pretrained)

    # ---- checkpoints (pipeline.py:66-83): the reference's four directories under `pretrained_weights/`
    @classmethod
    def _required_files(cls) -> list:
        """(subdirectory of the weights root, file names of which one must exist) for every model this pipeline loads."""
        from .background_removal import B200BackgroundRemover
        from .stage0 import TRIPOSG_FILES

        return ([(os.path.join("TripoSG", d), names) for d, names in TRIPOSG_FILES]
                + [("dinov2", ("config.json",)), ("dinov2", B200ImageEncoder.weight_files),
                   ("dinov2", ("preprocessor_config.json",)), ("RMBG", B200BackgroundRemover.weight_files)]
                + [(os.path.join("ActionMesh", d), names) for d in ("denoiser", "autoencoder")
                   for names in (("config.json",), B200Denoiser.weight_files)])

    @classmethod
    def from_pretrained(cls, weights_root: str = "pretrained_weights", config_name: str = "actionmesh_b200.yaml",
                        config_dir: Optional[str] = None, lazy_loading: bool = False, *, dtype: torch.dtype = torch.bfloat16,
                        config_updates: Optional[dict] = None):
        """The pipeline the reference builds, from the reference's checkpoint directories under `weights_root`: TripoSG
        (Stage 0), dinov2 (Stage I's image encoder, fp32-grade), RMBG (background removal) and ActionMesh (denoiser/,
        autoencoder/).  Frames are cropped by `B200FramePreprocessor` and the anchor mesh is post-processed by
        `B200MeshPostprocessor`.  Every required file is checked here, before any GPU work: a missing one raises an
        AmbError naming it.  Models are loaded by `.to(device)`, or with `lazy_loading` just before their stage and
        released right after it."""
        from .mesh_process import B200MeshPostprocessor
        from .module import check_files
        from .preprocess import B200FramePreprocessor

        check_files(weights_root, cls._required_files(), "ActionMesh checkpoints")
        target = f"{B200MeshPostprocessor.__module__}.{B200MeshPostprocessor.__name__}"
        pipe = cls(config_name, config_dir, dtype, lazy_loading, image_process=B200FramePreprocessor(),
                   weights_dir=os.path.join(weights_root, "ActionMesh"),
                   config_updates={"model.mesh_process._target_": target, **(config_updates or {})})
        pipe._bind_checkpoints(weights_root)
        return pipe

    def _bind_checkpoints(self, weights_root: str) -> None:
        """Loaders (callables, so that lazy loading never holds two large models at once) of the models that do not come
        from the ActionMesh directory."""
        from .background_removal import B200BackgroundRemover
        from .stage0 import TripoSGStage0

        dino = os.path.join(weights_root, "dinov2")
        self._loaders = {
            "background_removal": lambda: B200BackgroundRemover(os.path.join(weights_root, "RMBG")).to(self._target_device),
            "image_to_3d_pipe": lambda: TripoSGStage0.from_pretrained(os.path.join(weights_root, "TripoSG"),
                                                                      device=self._target_device,
                                                                      num_tokens=self._denoiser_latent_shape[0]),
            "image_encoder": lambda: B200ImageEncoder.from_hf_dirs(dino, dino, precision="fp32", device=self._target_device),
        }

    # ---- model lifecycle (pipeline.py:117-229)
    def _load_from_checkpoint(self, attr: str) -> None:
        """Build `attr` with its checkpoint loader when it is not loaded; an injected component is left as it is."""
        if getattr(self, attr) is None and attr in self._loaders:
            setattr(self, attr, self._loaders[attr]())

    def _release(self, attr: str) -> None:
        """`_unload_model` for a component `from_pretrained` can load again (an injected one is kept)."""
        if attr in self._loaders:
            self._unload_model(attr)

    def _load_image_to_3d(self) -> None:
        self._load_from_checkpoint("image_to_3d_pipe")

    def _load_background_removal(self) -> None:
        self._load_from_checkpoint("background_removal")

    def _load_image_encoder(self) -> None:
        self._load_from_checkpoint("image_encoder")
        if self.image_encoder is None:
            self.image_encoder = instantiate(self.cfg.model.image_encoder, _convert_="partial")()
        self.image_encoder.to(self._target_device)

    def _load_temporal_denoiser(self) -> None:
        if self.temporal_3D_denoiser is None:
            cls = get_target(self.cfg.model.temporal_3D_denoiser["_target_"])
            self.temporal_3D_denoiser = cls.from_pretrained(os.path.join(self._actionmesh_weights_dir, "denoiser"),
                                                            device=self._target_device)
        self.temporal_3D_denoiser.to(self._target_device)

    def _load_temporal_vae(self) -> None:
        if self.temporal_3D_vae is None:
            cls = get_target(self.cfg.model.temporal_3D_vae["_target_"])
            self.temporal_3D_vae = cls.from_pretrained(os.path.join(self._actionmesh_weights_dir, "autoencoder"),
                                                       device=self._target_device)
        self.temporal_3D_vae.to(self._target_device)

    def _unload_model(self, attr: str) -> None:
        if self._lazy_loading and getattr(self, attr, None) is not None:
            setattr(self, attr, None)
            torch.cuda.empty_cache()

    def to(self, device) -> "ActionMeshB200Pipeline":
        device = torch.device(device)
        if device.type != "cuda":
            raise AmbError("ActionMeshB200Pipeline runs on CUDA (sm_90a) only; there is no CPU fallback")
        self._target_device = device
        if not self._lazy_loading:
            self._load_background_removal()
            self._load_image_to_3d()
            self._load_image_encoder()
            self._load_temporal_denoiser()
            self._load_temporal_vae()
        return self

    @property
    def device(self) -> torch.device:
        return self._target_device

    # ---- stages
    def _apply_overrides(self, input, stage_0_steps, face_decimation, floaters_threshold, stage_1_steps, guidance_scales,
                         anchor_idx) -> None:
        """The per-call overrides of `__call__` (pipeline.py:637-656), then background removal and image processing of
        the frames."""
        if stage_0_steps is not None:
            self.cfg.model.image_to_3D_denoiser.num_inference_steps = stage_0_steps
        if stage_1_steps is not None:
            self.scheduler.num_inference_steps = stage_1_steps
        if guidance_scales is not None:
            self.cf_guidance.guidance_scales = guidance_scales
        if face_decimation is not None:
            self.mesh_process.face_decimation = face_decimation
        if floaters_threshold is not None:
            self.mesh_process.floaters_threshold = floaters_threshold
        if anchor_idx is not None:
            self.cfg.anchor_idx = anchor_idx
        self._load_background_removal()
        if self.background_removal is not None:
            input.frames = self.background_removal.process_images(input.frames)
        self._release("background_removal")
        if self.image_process is not None:
            input.frames = self.image_process.process_images(input.frames)

    def init_banks_from_anchor(self, input, seed: int = 44):
        """Stage 0 through the injected image-to-3D component (pipeline.py:387-433) -> (LatentBank, anchor mesh)."""
        if self.image_to_3d_pipe is None:
            raise AmbError("no Stage 0 (TripoSG image-to-3D): build the pipeline with from_pretrained(weights_root) or pass "
                           "image_to_3d=<callable> returning (anchor_latent, anchor_mesh)")
        gen_dev = getattr(self.image_to_3d_pipe, "device", self._target_device)
        anchor_latent, anchor_mesh = self.image_to_3d_pipe(
            image=input.frames[self.cfg.anchor_idx], generator=torch.Generator(device=gen_dev).manual_seed(seed),
            num_inference_steps=self.cfg.model.image_to_3D_denoiser.num_inference_steps,
            guidance_scale=self.cfg.model.image_to_3D_denoiser.guidance_scale)
        anchor_mesh = self.mesh_process.process_mesh(anchor_mesh, seed=seed)
        bank = LatentBank(empty_dims=self._denoiser_latent_shape)
        bank.update(timesteps=input.timesteps[[self.cfg.anchor_idx]],
                    latents=torch.as_tensor(anchor_latent).to(device=self._target_device, dtype=torch.float32))
        return bank, anchor_mesh

    def _stage_pipeline(self) -> "AnimationPipeline":
        faces_holder = {}
        normals_fn = lambda verts: vertex_normals(verts, faces_holder["faces"])
        pipe = AnimationPipeline(self.temporal_3D_denoiser, self.scheduler, self.cf_guidance, self.temporal_3D_vae,
                                 self.image_encoder, sliding_window_autoencoder=self.cfg.sliding_window_autoencoder,
                                 subsampling_level=self.cfg.subsampling_level, normals_fn=normals_fn,
                                 temporal_context_size=self.cfg.model.temporal_3D_denoiser.temporal_context_size,
                                 sliding_window_denoiser=self.cfg.sliding_window_denoiser, anchor_idx=self.cfg.anchor_idx,
                                 latent_shape=self._denoiser_latent_shape)
        pipe._faces_holder = faces_holder
        return pipe

    @torch.no_grad()
    def __call__(self, input, seed: int = 44, stage_0_steps: Optional[int] = None, face_decimation: Optional[int] = None,
                 floaters_threshold: Optional[float] = None, stage_1_steps: Optional[int] = None,
                 guidance_scales: Optional[List[float]] = None, anchor_idx: Optional[int] = None) -> list:
        """video -> 4D (pipeline.py:602-685): returns the animated meshes (fixed topology) ordered by timestep."""
        self._apply_overrides(input, stage_0_steps, face_decimation, floaters_threshold, stage_1_steps, guidance_scales,
                              anchor_idx)
        self._load_image_to_3d()
        latent_bank, anchor_mesh = self.init_banks_from_anchor(input, seed)          # Stage 0
        self._release("image_to_3d_pipe")
        ordered = self._animate(input, latent_bank, anchor_mesh.vertices, anchor_mesh.faces, anchor_mesh.vertex_normals, seed)
        f_np = torch.as_tensor(anchor_mesh.faces).to(torch.int64).numpy()
        return [_make_output_mesh(v.cpu().numpy(), f_np) for v in ordered]

    def _animate(self, input, latent_bank: LatentBank, vertices, faces, vertex_normals, seed: int) -> list:
        """DinoV2 on all frames, Stage I from the seeded `latent_bank`, then Stage II from the anchor mesh -> the (V, 3)
        vertex tensors of every output timestep, in order."""
        self._load_image_encoder()
        vin = VideoInput(list(input.frames), input.timesteps)
        self._load_temporal_denoiser()
        self._load_temporal_vae()
        stages = self._stage_pipeline()
        context = stages.encode_all_frames(vin)                                       # DinoV2 on all frames
        self._unload_model("image_encoder")
        latent_bank = stages.generate_3d_latents(vin, context, latent_bank, seed=seed)   # Stage I
        self._unload_model("temporal_3D_denoiser")
        dev = self._target_device
        verts = torch.as_tensor(vertices, dtype=torch.float32).to(dev)
        faces = torch.as_tensor(faces).to(torch.int64)
        normals = torch.as_tensor(vertex_normals, dtype=torch.float32).to(dev)
        stages._faces_holder["faces"] = faces
        vb = VertexBank(faces=faces)
        vb.update(timesteps=input.timesteps[[self.cfg.anchor_idx]], vertices=[verts])
        vb = stages.generate_mesh_animation(latent_bank, vb, normals)               # Stage II
        self._unload_model("temporal_3D_vae")
        ordered, _ = vb.get_ordered()
        return ordered


def _make_output_mesh(vertices, faces):
    """trimesh.Trimesh(vertices, faces, process=False) as the reference returns, or the package's `Mesh`."""
    try:
        import trimesh

        return trimesh.Trimesh(vertices=vertices, faces=faces, process=False)
    except ImportError:
        return Mesh(vertices=vertices, faces=faces)


class ActionMeshB200PipelineWithMeshInput(ActionMeshB200Pipeline):
    """{video + 3D mesh} -> 4D: `ActionMeshPipelineWithMeshInput` (reference actionmesh/pipeline_with_3d.py:27-240) on the
    CUDA path.  The user's mesh is merged and cleaned, normalized, sampled (16384 surface points with face normals) and
    encoded by the TripoSG VAE encoder (`B200TripoSGVAE.encode_to_latent`) into the anchor latent; Stage I and Stage II are
    the base pipeline's.  The outputs are denormalized and expanded back to the input's own vertices and faces
    (`pre_merge_faces`), so its UVs and textures still apply.  No mesh post-processing runs on this path, as in the reference.

    The VAE is `B200TripoSGVAE.from_pretrained(f"{triposg_weights_dir}/vae")`, or assigned directly (`pipe.vae = model`).
    Unlike the reference, which passes no seed to the encoder's point sampling and posterior sample, both are seeded from
    `seed`, so two calls with the same seed give the same meshes.  Like the reference, `anchor_mesh` is modified in place."""

    def __init__(self, *args, triposg_weights_dir: str = "pretrained_weights/TripoSG", **kwargs):
        super().__init__(*args, **kwargs)
        self._triposg_weights_dir = triposg_weights_dir
        self.vae = None

    @classmethod
    def _required_files(cls) -> list:
        """The base pipeline's files, with TripoSG's VAE in place of the whole of Stage 0."""
        from .triposg_vae import B200TripoSGVAE

        vae = os.path.join("TripoSG", "vae")
        return ([(vae, ("config.json",)), (vae, B200TripoSGVAE.weight_files)]
                + [e for e in super()._required_files() if not e[0].startswith("TripoSG")])

    def _bind_checkpoints(self, weights_root: str) -> None:
        super()._bind_checkpoints(weights_root)
        del self._loaders["image_to_3d_pipe"]
        self._triposg_weights_dir = os.path.join(weights_root, "TripoSG")

    def _load_vae(self) -> None:
        if self.vae is None:
            from .triposg_vae import B200TripoSGVAE

            self.vae = B200TripoSGVAE.from_pretrained(os.path.join(self._triposg_weights_dir, "vae"), device=self._target_device)
        self.vae.to(self._target_device)

    def to(self, device) -> "ActionMeshB200PipelineWithMeshInput":
        super().to(device)
        if not self._lazy_loading:
            self._load_vae()
        return self

    def init_banks_from_anchor(self, input, anchor_mesh, seed: int = 44):
        """pipeline_with_3d.py:60-125 -> (latent_bank, vertex_bank, normalization, vertex_merge_map, pre_merge_faces).
        `vertex_bank` holds the merged, normalized anchor vertices at the anchor timestep (its `faces` the merged faces):
        the vertex-only counterpart of the reference's MeshBank."""
        from .mesh_input import merge_and_clean_mesh, normalize_mesh, sample_surface

        vertex_merge_map, pre_merge_faces = merge_and_clean_mesh(anchor_mesh)
        anchor_mesh, params = normalize_mesh(anchor_mesh)
        surface = sample_surface(anchor_mesh, n_points=16384, seed=seed, with_normals=True, device=self._target_device,
                                 dtype=torch.float32)
        anchor_latent = self.vae.encode_to_latent(surface, seed=seed, generator=torch.Generator().manual_seed(seed))
        anchor_t = input.timesteps[[self.cfg.anchor_idx]]
        latent_bank = LatentBank(empty_dims=self._denoiser_latent_shape)
        latent_bank.update(timesteps=anchor_t, latents=anchor_latent.to(dtype=torch.float32))
        faces = torch.as_tensor(anchor_mesh.faces).to(torch.int64)
        vertex_bank = VertexBank(faces=faces)
        vertex_bank.update(timesteps=anchor_t, vertices=[torch.as_tensor(anchor_mesh.vertices, dtype=torch.float32)])
        return latent_bank, vertex_bank, params, vertex_merge_map, pre_merge_faces

    @torch.no_grad()
    def __call__(self, input, anchor_mesh, seed: int = 44, stage_0_steps: Optional[int] = None,
                 face_decimation: Optional[int] = None, floaters_threshold: Optional[float] = None,
                 stage_1_steps: Optional[int] = None, guidance_scales: Optional[List[float]] = None,
                 anchor_idx: Optional[int] = None) -> list:
        """{video + 3D mesh} -> 4D (pipeline_with_3d.py:127-240): the animated meshes with the input mesh's own vertices
        and faces, ordered by timestep."""
        from .mesh_input import denormalize_mesh

        self._apply_overrides(input, stage_0_steps, face_decimation, floaters_threshold, stage_1_steps, guidance_scales,
                              anchor_idx)
        self._load_vae()
        latent_bank, vertex_bank, params, vertex_merge_map, pre_merge_faces = self.init_banks_from_anchor(input, anchor_mesh, seed)
        self._unload_model("vae")
        verts = vertex_bank.get(timesteps=input.timesteps[[self.cfg.anchor_idx]])[0]
        faces = vertex_bank.faces
        ordered = self._animate(input, latent_bank, verts, faces, vertex_normals(verts, faces), seed)
        out = []
        for v in ordered:
            m = denormalize_mesh(Mesh(vertices=v.cpu().numpy().astype(np.float64), faces=None), params)
            out.append(_make_output_mesh(np.asarray(m.vertices)[vertex_merge_map], pre_merge_faces))
        return out
