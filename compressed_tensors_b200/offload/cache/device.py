"""`DeviceCache`: offloaded tensors stay in device memory (`offload_device`, by default the onload device); onloading only moves
them when the onload device was changed after the module was offloaded."""
from __future__ import annotations

from typing import Literal

import torch

from ..utils import send_tensors
from .base import OffloadCache

__all__ = ["DeviceCache"]


class DeviceCache(OffloadCache):
    def __init__(self, onload_device: torch.device | str, offload_device: torch.device | str | Literal["disk"] | None = None):
        super().__init__(onload_device, offload_device=offload_device)
        self.offload_device = torch.device(offload_device) if offload_device is not None else self.onload_device

    def onload(self, offloaded: torch.Tensor | None) -> torch.Tensor | None:
        return send_tensors(offloaded, device=self.onload_device, copy=False)

    def offload(self, tensor: torch.Tensor | None) -> torch.Tensor | None:
        return send_tensors(tensor, device=self.offload_device, copy=False)

    @torch.no_grad()
    def update_offload(self, offloaded: torch.Tensor, data: torch.Tensor | None):
        if data is not None:
            offloaded.copy_(data)
