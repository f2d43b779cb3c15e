"""Stage 0 on the CUDA path — SURVEY 8(f) rank 2: TripoSG's DiT denoising loop, the step that produces the anchor latent
(reference actionmesh/pipeline.py:387-433 -> third_party/TripoSG).

TripoSG's DiT (triposg/models/transformers/triposg_transformer.py:129-362,365-726) is the block family ActionMesh's
denoiser derives from: the forward of ONE frame without rotary embedding, same time token, same head-interleaved q/k/v
split, same long skips.  `B200TripoSGDiT` therefore is the `B200Denoiser` launch program at T = 1 behind TripoSGDiTModel's
`forward(hidden_states, timestep, encoder_hidden_states, return_dict)` and state-dict keys; `B200RectifiedFlowScheduler`
mirrors `RectifiedFlowScheduler.set_timesteps / step` (triposg/schedulers/scheduling_rectified_flow.py:177-215,234-308);
`TripoSGStage0.denoise` is the loop of `TripoSGPipeline.__call__` (triposg/pipelines/pipeline_triposg.py:243-294) with the
CFG combine + Euler update fused in one kernel (amb_cfg_euler_step) and the zero-embedding branch's cross-attention folded
to its bias (SURVEY A.5).

Precision: the reference runs this stage in fp16 (pipeline.py:142); here GEMM / attention operands are bf16 with fp32
accumulation and an fp32 residual stream, latents stay fp32 between steps (the reference rounds them to fp16 every step,
scheduling_rectified_flow.py:299).  tests/test_stage0_gpu.py states the tolerance against the fp32 reference modules.
The VAE decoder and the iso-surface extraction that turn the latent into the anchor MESH live in triposg_vae.py:
`TripoSGStage0(..., mesh_extractor=B200TripoSGVAE.extract_mesh)` (bound to a loaded VAE).  Without an extractor,
`__call__` raises.  `TripoSGStage0.from_pretrained(triposg_dir)` builds the DiT, the VAE, TripoSG's DinoV2 and the
scheduler shift from the reference's TripoSG checkpoint directory (DESIGN section 18).
"""
from __future__ import annotations

import json
import os
from typing import Callable, Optional

import numpy as np
import torch

from ._lib import AmbError
from .blocks import remap_triposg_state_dict
from .denoiser import B200Denoiser, DenoiserConfig
from .guidance import ClassifierFreeGuidance
from .image_encoder import B200ImageEncoder
from .module import check_files
from .scheduler import B200SchedulerFlow
from .triposg_vae import B200TripoSGVAE


class B200TripoSGDiT(B200Denoiser):
    """Drop-in for TripoSGDiTModel on the denoising path: constructor arguments of triposg_transformer.py:412-421, and
    `from_pretrained` of a diffusers directory (config.json + diffusion_pytorch_model.safetensors)."""

    config_class = None
    weight_files = ("diffusion_pytorch_model.safetensors", "diffusion_pytorch_model.bin")

    def __init__(self, num_attention_heads: int = 16, width: int = 2048, in_channels: int = 64, num_layers: int = 21,
                 cross_attention_dim: int = 1024, **kwargs):
        if kwargs.get("use_cross_attention_2"):
            raise AmbError("B200TripoSGDiT: the second cross-attention branch is not used by ActionMesh's Stage 0")
        super().__init__(DenoiserConfig(num_tokens_nominal=2048, temporal_context_size=1, in_channels=in_channels,
                                        num_layers=num_layers, num_attention_heads=num_attention_heads, width=width,
                                        cross_attention_dim=cross_attention_dim, inflated_layers=()))

    def _pack_state_dict(self, sd: dict, dev: torch.device) -> dict:
        return super()._pack_state_dict(remap_triposg_state_dict(sd), dev)

    @torch.no_grad()
    def forward(self, hidden_states: torch.Tensor, timestep: torch.Tensor, encoder_hidden_states: torch.Tensor = None,
                attention_kwargs=None, return_dict: bool = True):
        """(B, N, C), (B,), (B, S, Dc) -> (B, N, C) bf16 [a 1-tuple like the reference when return_dict=False]."""
        B = hidden_states.shape[0]
        t = timestep if torch.is_tensor(timestep) else torch.tensor([float(timestep)])
        out, _ = B200Denoiser.forward(self, hidden_states[:, None], encoder_hidden_states[:, None], torch.zeros(B, 1),
                                      t.reshape(-1).expand(B), None, None)
        out = out[:, 0]
        return (out,) if not return_dict else out

    __call__ = forward


class B200RectifiedFlowScheduler:
    """RectifiedFlowScheduler (scheduling_rectified_flow.py:78-308): same constructor arguments, `set_timesteps`, `timesteps`,
    `sigmas`, `step(model_output, timestep, sample, return_dict)`.  `step` keeps the sample in fp32."""

    order = 1

    def __init__(self, num_train_timesteps: int = 1000, shift: float = 1.0, use_dynamic_shifting: bool = False):
        if use_dynamic_shifting:
            raise AmbError("dynamic shifting is not used by ActionMesh's Stage 0")
        self.num_train_timesteps, self.shift = num_train_timesteps, shift
        self.timesteps = self.sigmas = None
        self._step_index = None

    def set_timesteps(self, num_inference_steps: int, device=None, sigmas=None, mu=None) -> None:
        n = self.num_train_timesteps
        if sigmas is None:
            self.num_inference_steps = num_inference_steps
            sigmas = np.array([(1.0 - i / num_inference_steps) * n for i in range(num_inference_steps)]) / n
        sigmas = self.shift * np.asarray(sigmas) / (1 + (self.shift - 1) * np.asarray(sigmas))
        sig = torch.from_numpy(sigmas).to(torch.float32)
        self.timesteps = (sig * n).to(device) if device is not None else sig * n
        self.sigmas = torch.cat([sig, torch.zeros(1)])  # host side, like the reference (scheduling_rectified_flow.py:126)
        self._step_index = None

    @property
    def step_index(self):
        return self._step_index

    def step(self, model_output: torch.Tensor, timestep, sample: torch.Tensor, return_dict: bool = True, **unused):
        """x_{t-1} = x_t + (sigma_t - sigma_{t-1}) v  (scheduling_rectified_flow.py:283-305)."""
        if isinstance(timestep, int):
            raise ValueError("pass one of `scheduler.timesteps`, not an index")
        if self._step_index is None:
            hits = (self.timesteps.cpu() == float(timestep)).nonzero()
            self._step_index = int(hits[1 if len(hits) > 1 else 0])
        d = float(self.sigmas[self._step_index] - self.sigmas[self._step_index + 1])
        prev = sample.to(torch.float32) + d * model_output.to(torch.float32)
        self._step_index += 1
        return (prev,) if not return_dict else prev


class _Stage0Flow(B200SchedulerFlow):
    """The fused CFG + Euler loop of B200SchedulerFlow on the rectified-flow schedule: timesteps sigma_i * 1000 (+ the
    trailing 0), steps (sigma_i - sigma_{i+1})."""

    def get_schedule(self):
        rf = B200RectifiedFlowScheduler(self.num_train_timesteps, self.shift)
        rf.set_timesteps(self.num_inference_steps)
        return torch.cat([rf.timesteps, torch.zeros(1)]), rf.sigmas[:-1] - rf.sigmas[1:]


def scheduler_shift(scheduler_dir: str) -> float:
    """The `shift` of a diffusers `RectifiedFlowScheduler` directory (scheduler_config.json)."""
    path = os.path.join(scheduler_dir, "scheduler_config.json")
    if not os.path.isfile(path):
        raise AmbError(f"TripoSG scheduler: {path} not found")
    with open(path) as f:
        cfg = json.load(f)
    if cfg.get("use_dynamic_shifting", False):
        raise AmbError("dynamic shifting is not used by ActionMesh's Stage 0")
    if int(cfg.get("num_train_timesteps", 1000)) != 1000:
        raise AmbError(f"TripoSG scheduler: num_train_timesteps {cfg['num_train_timesteps']} (expected 1000)")
    return float(cfg.get("shift", 1.0))


# Subfolders of the TripoSG checkpoint (diffusers layout) and the files each one must hold (one of each tuple).
TRIPOSG_FILES = (("transformer", ("config.json",)), ("transformer", B200TripoSGDiT.weight_files),
                 ("vae", ("config.json",)), ("vae", B200TripoSGVAE.weight_files),
                 ("image_encoder_dinov2", ("config.json",)), ("image_encoder_dinov2", B200ImageEncoder.weight_files),
                 ("feature_extractor_dinov2", ("preprocessor_config.json",)), ("scheduler", ("scheduler_config.json",)))


class TripoSGStage0:
    """`image_to_3d` component of ActionMeshB200Pipeline: (image, generator, num_inference_steps, guidance_scale) ->
    (anchor_latent (1, N, C) fp32, anchor_mesh), as `TripoSGPipelinePlus.__call__` (actionmesh/external/triposg.py:35).

    `image_encoder`: B200ImageEncoder with TripoSG's DinoV2 weights (pipeline_triposg.py:137-145); `mesh_extractor(latents)`:
    the VAE decode + iso-surface extraction, e.g. `B200TripoSGVAE(...).extract_mesh` (triposg_vae.py).
    `from_pretrained(triposg_dir)` builds all of it from the TripoSG checkpoint directory."""

    def __init__(self, transformer: B200TripoSGDiT, image_encoder, mesh_extractor: Optional[Callable] = None,
                 shift: float = 1.0, num_tokens: int = 2048):
        self.transformer, self.image_encoder, self.mesh_extractor = transformer, image_encoder, mesh_extractor
        self.shift, self.num_tokens = shift, num_tokens

    @classmethod
    def from_pretrained(cls, triposg_dir: str, device="cuda", num_tokens: int = 2048) -> "TripoSGStage0":
        """The TripoSG checkpoint directory (diffusers layout: transformer/, vae/, image_encoder_dinov2/,
        feature_extractor_dinov2/, scheduler/) -> Stage 0 on `device`, with the VAE's `extract_mesh` at the defaults of
        `TripoSGPipelinePlus.__call__` (bounds +-1.005, octree depth 9) as the mesh extractor.

        TripoSG's DinoV2 runs with bf16 operands: the reference casts the whole TripoSG pipeline to fp16, and this package
        uses bf16 where the reference uses fp16 in Stage 0 (DESIGN section 11).  bf16 also puts its attention on the wgmma
        flash-attention kernel, which takes any sequence length, whatever crop the feature extractor asks for."""
        check_files(triposg_dir, TRIPOSG_FILES, "TripoSG checkpoint")
        shift = scheduler_shift(os.path.join(triposg_dir, "scheduler"))
        transformer = B200TripoSGDiT.from_pretrained(os.path.join(triposg_dir, "transformer"), device=device)
        vae = B200TripoSGVAE.from_pretrained(os.path.join(triposg_dir, "vae"), device=device)
        encoder = B200ImageEncoder.from_hf_dirs(os.path.join(triposg_dir, "image_encoder_dinov2"),
                                                os.path.join(triposg_dir, "feature_extractor_dinov2"), precision="bf16",
                                                device=device)
        return cls(transformer, encoder, mesh_extractor=vae.extract_mesh, shift=shift, num_tokens=num_tokens)

    @property
    def device(self) -> torch.device:
        return self.transformer.device

    @torch.no_grad()
    def denoise(self, image_embeds: torch.Tensor, latents: torch.Tensor, num_inference_steps: int = 50,
                guidance_scale: float = 7.0) -> torch.Tensor:
        """(1, S, Dc) embeddings, (1, N, C) initial noise -> denoised (1, N, C) fp32 latents."""
        dev = self.device
        cf = ClassifierFreeGuidance(inference_enabled=guidance_scale > 1, guidance_at_inference=[[0, 1], [1, 1]],
                                    guidance_scales=[float(guidance_scale)])
        flow = _Stage0Flow(num_inference_steps=num_inference_steps, shift=self.shift, is_additive=True)
        x = latents.to(device=dev, dtype=torch.float32)[:, None].contiguous()       # one "frame"
        out = flow.denoise(self.transformer, cf, x, image_embeds.to(dev)[:, None], device=dev, mask=None,
                           framestep=torch.zeros(1, 1))
        return out[:, 0]

    @torch.no_grad()
    def __call__(self, image, generator=None, num_inference_steps: int = 50, guidance_scale: float = 7.0,
                 latents: Optional[torch.Tensor] = None):
        embeds = self.image_encoder.encode_images([image]) if not torch.is_tensor(image) else image
        c = self.transformer.config
        if latents is None:  # prepare_latents (pipeline_triposg.py:147-173): torch's generator for seed parity
            latents = torch.randn((1, self.num_tokens, c.in_channels), generator=generator,
                                  device=generator.device if generator is not None else self.device)
        lat = self.denoise(embeds.reshape(1, -1, embeds.shape[-1]), latents, num_inference_steps, guidance_scale)
        if self.mesh_extractor is None:
            raise AmbError("TripoSGStage0: no mesh extractor — pass mesh_extractor=<callable latents -> mesh> (e.g. "
                           "B200TripoSGVAE.extract_mesh) or build it with TripoSGStage0.from_pretrained")
        return lat, self.mesh_extractor(lat)
