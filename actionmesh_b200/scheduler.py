"""B200SchedulerFlow — flow-matching sampler with the reference's public surface (actionmesh/scheduler/scheduler.py).

Same dataclass fields and the `get_schedule / get_noise / denoise` signatures `ActionMeshPipeline._denoise_latents`
calls (pipeline.py:288,302), so the hydra `_target_` of `model.scheduler` can simply be re-pointed at this class.
What changes underneath when the model is a `B200Denoiser`:
  * the CFG batch is never concatenated: both branches read the same bf16 latents, the zero-image-context branch is
    known per window (no `zeros_like` + `cat` of 34 MB per step, guidance.py:56-91);
  * CFG combine + Euler step + observed-frame mask is ONE coalesced kernel writing the fp32 latents in place
    (amb_cfg_euler_step), with no `assert unobserved.any()` device->host sync per step (scheduler.py:245);
  * RoPE tables and the context K/V of all layers are computed once per window (WindowState).
`step()` exposes the fused update on its own (the reference has no step(); SURVEY D1).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Callable, Optional

import numpy as np
import torch

from . import ops
from ._lib import AmbError
from .denoiser import B200Denoiser, WindowState
from .guidance import ClassifierFreeGuidance


@dataclass(eq=False)
class B200SchedulerFlow:
    """Flow-matching scheduler (fields as SchedulerFlow, scheduler.py:24-41)."""

    num_inference_steps: int
    num_train_timesteps: int = 1000
    shift: float = 3.0
    is_additive: bool = False
    split_cfg_batch: bool = False  # accepted for config compatibility; the CUDA path never needs the split

    # ---------------------------------------------------------------- schedule (host, float64 -> float32)
    def get_schedule(self) -> tuple[torch.Tensor, torch.Tensor]:
        timesteps = self._compute_timesteps(self.num_inference_steps + 1, self.num_train_timesteps, self.shift)
        distances = (timesteps[:-1] - timesteps[1:]) / self.num_train_timesteps
        return timesteps, distances

    @staticmethod
    def _compute_timesteps(num_inference_steps: int, num_train_timesteps: int = 1000, shift: float = 1.0) -> torch.Tensor:
        """sigma(u) = s u / (1 + (s-1) u) on u = linspace(1, sigma_min); sigma_min = shifted 1/N (scheduler.py:59-98)."""
        n = num_train_timesteps
        lo = shift * (1.0 / n) / (1 + (shift - 1) * (1.0 / n))
        u = np.linspace(1.0 * n, lo * n, num_inference_steps) / n
        sig = shift * u / (1 + (shift - 1) * u)
        return torch.from_numpy((sig * n).astype(np.float32))

    # ---------------------------------------------------------------- noise (torch Philox, kept for seed parity; SURVEY A.6)
    def get_noise(self, latent_shape, batch_size: int, n_timesteps: int, device, generator=None,
                  corr_noise: float = 0.0) -> torch.Tensor:
        assert 0 <= corr_noise <= 1.0
        same = torch.randn([batch_size, 1] + list(latent_shape), generator=generator, device=device)
        indep = torch.randn([batch_size, n_timesteps] + list(latent_shape), generator=generator, device=device)
        if corr_noise == 0.0:
            return indep  # the shared draw still advanced the generator, as in the reference
        return math.sqrt(corr_noise) * same.repeat(1, n_timesteps, 1, 1) + math.sqrt(1 - corr_noise) * indep

    # ---------------------------------------------------------------- fused update, usable on its own
    def step(self, model_output: torch.Tensor, step_index: int, sample: torch.Tensor,
             mask: Optional[torch.Tensor] = None, guidance_scales: Optional[list] = None) -> torch.Tensor:
        """x <- x ± distances[i] * cfg(model_output) on unobserved frames, in place (scheduler.py:238-248).

        model_output: (K*B, T, N, C) bf16 contiguous CFG-stacked predictions; sample: (B, T, N, C) fp32 CUDA."""
        _, distances = self.get_schedule()
        B, T, N, C = sample.shape
        K = model_output.shape[0] // B
        upd = torch.ones(B * T, dtype=torch.uint8, device=sample.device) if mask is None else \
            (mask.reshape(B * T) == 0).to(torch.uint8)
        dt = float(distances[step_index]) * (1.0 if self.is_additive else -1.0)
        mo = model_output.contiguous()
        ops.cfg_euler_step(sample, mo, list(guidance_scales or []), dt, upd, n_branches=K,
                           branch_stride=B * T * N * C, frame_stride=N * C, frame_offset=0, n_per_frame=N * C)
        return sample

    # ---------------------------------------------------------------- denoise loop
    @torch.no_grad()
    def denoise(self, diffusion_model, cf_guidance: ClassifierFreeGuidance, init_latent: torch.Tensor,
                context: torch.Tensor, device="cuda:0", disable_prog: bool = True,
                mask: Optional[torch.Tensor] = None, framestep: Optional[torch.Tensor] = None,
                step_callback: Optional[Callable] = None, shard=None) -> torch.Tensor:
        """Same contract as SchedulerFlow.denoise (scheduler.py:253-295): returns the denoised latents; `init_latent`
        is updated in place on unobserved frames and observed frames stay bit-identical.

        `shard` (window_shard.FrameShard, optional extension): every rank calls denoise() with the SAME full-window
        arguments; each rank denoises its own frames (K/V all-gathered per layer) and the result is all-gathered."""
        if not isinstance(diffusion_model, B200Denoiser):
            raise AmbError("B200SchedulerFlow.denoise drives a B200Denoiser (no CPU / generic-module fallback)")
        model = diffusion_model
        if init_latent.dtype != torch.float32 or not init_latent.is_cuda:
            raise AmbError("init_latent must be an fp32 CUDA tensor")
        if init_latent.device != model.device:
            raise AmbError(f"init_latent lives on {init_latent.device}, the model on {model.device}")
        with torch.cuda.device(init_latent.device):  # the C ABI launches on the current device
            return self._denoise(model, cf_guidance, init_latent, context, mask, framestep, step_callback, shard)

    def _denoise(self, model, cf_guidance, init_latent, context, mask, framestep, step_callback, shard):
        latents = init_latent if init_latent.is_contiguous() else init_latent.contiguous()
        if mask is not None and not bool((mask == 0).any()):  # scheduler.py:245 asserts this every step; once is enough
            raise AssertionError("No unobserved frames found")
        fsl = None
        if shard is not None and shard.world > 1:
            fsl = shard.frames(latents.shape[1])
            latents = latents[:, fsl].contiguous()
            mask = None if mask is None else mask.reshape(init_latent.shape[0], -1)[:, fsl]
        B, T, N, C = latents.shape
        timesteps, distances = self.get_schedule()
        branches = cf_guidance.branches()
        scales = list(cf_guidance.guidance_scales) if cf_guidance.inference_enabled else []
        K = len(branches)
        dev = latents.device

        # ---- per-window, step-invariant state
        ctx = context.to(device=dev, dtype=torch.float32)
        ctx_all = torch.cat([ctx if ui else torch.zeros_like(ctx) for ui, _ in branches], dim=0)  # once per window
        fs = framestep if framestep is not None else torch.zeros(B, ctx.shape[1])
        fs_all = torch.cat([fs] * K, dim=0)
        state: WindowState = model.precompute_window(ctx_all, fs_all, N, frame_slice=fsl)
        del ctx_all
        m32 = None
        upd = torch.ones(B * T, dtype=torch.uint8, device=dev)
        if mask is not None:
            mk = mask.to(device=dev, dtype=torch.float32).reshape(B, T)
            m32 = torch.cat([mk if ul else torch.zeros_like(mk) for _, ul in branches], dim=0).reshape(K * B * T).contiguous()
            upd = (mk.reshape(B * T) == 0).to(torch.uint8)
        ws = model._workspace(K * B, T, N, world=shard.world if fsl is not None else 1,
                              slot=getattr(shard, "slot", 0) if fsl is not None else 0,
                              shard=shard if fsl is not None else None)
        L = N + 1
        sign = 1.0 if self.is_additive else -1.0
        t_dev = timesteps.to(dev)
        for i in range(self.num_inference_steps):
            ops.cast_bf16(latents.view(B * T * N, C), out=ws["x_in"][: B * T * N])
            pred = model._forward_packed(ws, state, K * B, T, N, t_dev[i:i + 1], m32, n_input_branches=B,
                                         shard=shard if fsl is not None else None)
            ops.cfg_euler_step(latents, pred, scales, sign * float(distances[i]), upd, n_branches=K,
                               branch_stride=B * T * L * C, frame_stride=L * C, frame_offset=C, n_per_frame=N * C)
            if step_callback is not None:
                step_callback(i + 1, self.num_inference_steps)
        if fsl is not None:
            init_latent.copy_(shard.gather_latents(latents))  # once per window; observed frames come back unchanged
        elif latents.data_ptr() != init_latent.data_ptr():
            init_latent.copy_(latents)
        return init_latent
