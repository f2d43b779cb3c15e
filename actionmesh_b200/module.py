"""`B200Module`: the nn.Module-like surface every host-side model shares (`.device`, `.eval()`, `.to()`, `load_state_dict`,
`from_pretrained`), so device placement and checkpoint loading are decided in one place.

A model packs a state dict into kernel-ready tensors with `_pack_state_dict(sd, device)`, which runs under `device` and can
also run on the CPU (the launch-program tests pack that way); `load_state_dict` runs it on the model's CUDA device."""
from __future__ import annotations

import inspect
import json
import os

import torch

from ._lib import AmbError


def read_weights(path: str, names) -> dict:
    """The state dict in the first of the files `names` present in directory `path` (safetensors, or a torch.save)."""
    files = [os.path.join(path, n) for n in names]
    file = next((f for f in files if os.path.exists(f)), files[-1])
    if file.endswith(".safetensors"):
        from safetensors.torch import load_file

        return load_file(file)
    return torch.load(file, map_location="cpu")


def check_files(root: str, required, what: str) -> None:
    """`required`: (subdirectory, file names) pairs; each subdirectory of `root` must hold one of its names.  Raises one
    AmbError naming the first path that is missing (a subdirectory, or its preferred file name)."""
    for sub, names in required:
        d = os.path.join(root, sub)
        if not os.path.isdir(d):
            raise AmbError(f"{what}: directory {d} not found")
        if not any(os.path.isfile(os.path.join(d, n)) for n in names):
            raise AmbError(f"{what}: {os.path.join(d, names[0])} not found")


class B200Module:
    config_class = None                                        # dataclass whose fields the constructor's **kwargs take
    weight_files = ("model.safetensors", "pytorch_model.bin")  # in order of preference

    def __init__(self):
        self._device = torch.device("cpu")
        self._w: dict = {}          # packed device weights
        self._loaded = False

    @property
    def device(self) -> torch.device:
        return self._device

    def eval(self):
        return self

    def to(self, device):
        """Move to a CUDA device; `cuda` means the current device, so a later `torch.cuda.set_device` does not change
        which GPU the entry points run on."""
        device = torch.device(device)
        if device.type != "cuda":
            raise AmbError(f"{type(self).__name__} runs on CUDA (sm_90a) only; there is no CPU fallback")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        moved = device != self._device
        if self._loaded and moved:
            self._w = {k: v.to(device) for k, v in self._w.items()}
        self._device = device
        self._after_to(moved)
        return self

    def _after_to(self, moved: bool) -> None:
        """What a model does after `to()` beyond moving its packed weights."""

    def load_state_dict(self, sd: dict) -> None:
        if self._device.type != "cuda":
            raise AmbError("call .to('cuda') before load_state_dict")
        with torch.cuda.device(self._device):
            self._w = self._pack_state_dict(sd, self._device)
        self._loaded = True

    def _check_loaded(self) -> None:
        if not self._loaded:
            raise AmbError(f"{type(self).__name__}: weights not loaded")

    @classmethod
    def from_pretrained(cls, path: str, device="cuda"):
        """`path`/config.json (the keys the constructor accepts; absent: the defaults) and the first of `weight_files`
        present in `path`, loaded onto `device`."""
        kwargs = {}
        cfg_path = os.path.join(path, "config.json")
        if os.path.exists(cfg_path):
            with open(cfg_path) as f:
                raw = json.load(f)
            params = inspect.signature(cls).parameters
            keys = {n for n, p in params.items() if p.kind in (p.POSITIONAL_OR_KEYWORD, p.KEYWORD_ONLY)} - {"config"}
            if cls.config_class is not None:
                keys |= set(cls.config_class.__dataclass_fields__)
            kwargs = {k: (tuple(v) if isinstance(v, list) else v) for k, v in raw.items() if k in keys}
        model = cls(**kwargs).to(device)
        model.load_state_dict(read_weights(path, cls.weight_files))
        return model
