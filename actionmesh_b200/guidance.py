"""ClassifierFreeGuidance — same dataclass surface as the reference (actionmesh/scheduler/guidance.py:14-118).

`cfg_at_inference` / `aggregate_cfg` / `get_unobserved_mask` keep the reference's generic tensor semantics so any
duck-typed model works; the CUDA fast path in `B200SchedulerFlow` never materialises the CFG batch (the branches share
their latents) and fuses `aggregate_cfg` with the Euler update in one kernel (amb_cfg_euler_step).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Optional

import torch


@dataclass(eq=False)
class ClassifierFreeGuidance:
    """Conditioning order is [image conditioning | latent conditioning] (guidance.py:15-17)."""

    inference_enabled: bool = True
    guidance_at_inference: list = field(default_factory=lambda: [[0, 0], [0, 1], [1, 1]])
    guidance_scales: list = field(default_factory=lambda: [1.0, 1.0])

    def __post_init__(self):
        assert len(self.guidance_at_inference) == len(self.guidance_scales) + 1

    def branches(self) -> list[tuple[int, int]]:
        """[(use_image_context, use_latent_mask)] per CFG branch; a single all-on branch when guidance is disabled."""
        if not self.inference_enabled:
            return [(1, 1)]
        out = []
        for g in self.guidance_at_inference:
            g = list(g)
            if g not in ([0, 0], [0, 1], [1, 0], [1, 1]):
                raise Exception(f"Unknown guidance: {g}")
            out.append((int(g[0]), int(g[1])))
        return out

    def get_unobserved_mask(self, mask: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
        return None if mask is None else mask == 0

    def cfg_at_inference(self, latent, context, mask, framestep):
        """guidance.py:38-93: batch of K branches; image context and/or latent mask zeroed per branch."""
        if not self.inference_enabled:
            return latent, context, mask, framestep
        br = self.branches()
        latent = torch.cat([latent] * len(br))
        framestep = torch.cat([framestep] * len(br)) if framestep is not None else None
        ctx = torch.cat([context if ui else torch.zeros_like(context) for ui, _ in br], dim=0)
        msk = None
        if mask is not None:
            msk = torch.cat([mask if ul else torch.zeros_like(mask) for _, ul in br], dim=0)
        return latent, ctx, msk, framestep

    def aggregate_cfg(self, aggregated: torch.Tensor) -> torch.Tensor:
        """guidance.py:95-118: p0 + sum_i scale_i (p_{i+1} - p_i)."""
        if not self.inference_enabled:
            return aggregated
        parts = aggregated.chunk(len(self.guidance_at_inference), dim=0)
        assert len(parts) == len(self.guidance_at_inference), "Invalid guidance"
        out = parts[0]
        for i in range(len(parts) - 1):
            out = out + self.guidance_scales[i] * (parts[i + 1] - parts[i])
        return out
