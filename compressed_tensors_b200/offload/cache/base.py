"""
`OffloadCache`: the mapping that stands in for `module._parameters` / `module._buffers` of an offloaded module.

Assigning a tensor offloads it (to pinned host memory, to a safetensors file, or to a device); reading one onloads it to
`onload_device`.  Two class-wide switches change that:

  * `disable_offloading()`: the first read of a tensor keeps its onloaded copy (in `keep_onloaded_values`) and later reads
    return that same copy; the copies are released when the outermost context exits.
  * `disable_onloading()`: reads return the offloaded value itself and assignments store the value as given, with no device
    movement at all.  This is how the compressors read an offloaded model's host tensors without moving them.
"""
from __future__ import annotations

import contextlib
from abc import ABC, abstractmethod
from collections.abc import Hashable, MutableMapping
from typing import ClassVar, Literal

import torch

__all__ = ["OffloadCache"]


def _device_type(device) -> str:
    return "disk" if device == "disk" else torch.device(device).type


class OffloadCache(MutableMapping, ABC):
    onload_device: torch.device | str
    offload_device: torch.device | Literal["disk"]

    offloading_disabled: ClassVar[bool] = False
    onloading_disabled: ClassVar[bool] = False

    # offloaded tensor -> its onloaded copy, filled only while offloading is disabled (shared by every cache)
    keep_onloaded_values: ClassVar[dict[torch.Tensor, torch.Tensor]] = dict()

    # name -> offloaded tensor (or None)
    offloaded_values: dict[Hashable, torch.Tensor | None]

    @classmethod
    def cls_from_device(cls, device: torch.device | str | Literal["disk"] | None = None) -> type["OffloadCache"]:
        """the cache class that offloads to `device`: CPUCache for "cpu", DiskCache for "disk", DeviceCache for an accelerator"""
        from .cpu import CPUCache
        from .device import DeviceCache
        from .disk import DiskCache

        kind = _device_type(device)
        import torch.distributed as dist

        if dist.is_available() and dist.is_initialized():
            name = {"cpu": "DistributedCPUCache (offload/cache/dist_cpu)", "disk": "DistributedDiskCache (offload/cache/dist_disk)"}.get(
                kind, "DistributedDeviceCache (offload/cache/dist_device)")
            raise NotImplementedError(f"{name}: offloading under an initialised torch.distributed process group needs the distributed "
                                      "caches, which compressed_tensors_b200 does not implement (DESIGN.md section 7)")
        if kind == "cpu":
            return CPUCache
        if kind == "disk":
            return DiskCache
        if kind in ("cuda", "xpu", "mps", "hpu", "npu", "mtia"):
            return DeviceCache
        raise NotImplementedError(f"Offload of type {kind} has not been implemented")

    @classmethod
    def from_mapping(cls, mapping: MutableMapping[Hashable, torch.Tensor | None], onload_device: torch.device | str,
                     offload_device: torch.device | str | Literal["disk"] | None = None, **kwargs) -> "OffloadCache":
        """a cache holding every value of `mapping` (typically a module's `_parameters` or `_buffers`), offloaded"""
        cache = cls(onload_device=onload_device, offload_device=offload_device, **kwargs)
        cache.offloaded_values = {name: cache.offload(value) for name, value in mapping.items()}
        return cache

    def __init__(self, onload_device: torch.device | str, offload_device: torch.device | str | Literal["disk"] | None = None):
        super().__init__()
        self.onload_device = onload_device
        self.offloaded_values = dict()
        # caches with a fixed offload device (CPU, disk) only accept that device
        if offload_device is not None and hasattr(type(self), "offload_device"):
            assert str(offload_device) == str(type(self).offload_device), f"{type(self).__name__} offloads to {type(self).offload_device}"

    @abstractmethod
    def onload(self, offloaded: torch.Tensor | None) -> torch.Tensor | None:
        """the offloaded tensor, brought to `onload_device`"""

    @abstractmethod
    def offload(self, tensor: torch.Tensor | None) -> torch.Tensor | None:
        """the tensor, moved to where this cache keeps its values; returns what goes into `offloaded_values`"""

    @abstractmethod
    def update_offload(self, offloaded: torch.Tensor, data: torch.Tensor | None):
        """overwrite the offloaded tensor's data in place with `data` (same shape)"""

    def __getitem__(self, key: Hashable) -> torch.Tensor | None:
        offloaded = self.offloaded_values[key]
        if offloaded is None or OffloadCache.onloading_disabled:
            return offloaded
        kept = OffloadCache.keep_onloaded_values.get(offloaded, None)
        if kept is not None:
            return kept
        onloaded = self.onload(offloaded)
        if OffloadCache.offloading_disabled:
            OffloadCache.keep_onloaded_values[offloaded] = onloaded
        return onloaded

    def __setitem__(self, key: Hashable, value: torch.Tensor | None):
        if OffloadCache.onloading_disabled:
            self.offloaded_values[key] = value
            return
        offloaded = self.offloaded_values.get(key, None)
        if offloaded is not None and value is not None and torch.is_same_size(offloaded, value):
            # same shape: write into the existing offloaded tensor, and into its kept onloaded copy if there is one
            self.update_offload(offloaded, value)
            kept = OffloadCache.keep_onloaded_values.get(offloaded, None)
            if kept is not None and kept is not offloaded:
                with torch.no_grad():
                    kept.copy_(value)
        else:
            self.offloaded_values[key] = self.offload(value)

    def __delitem__(self, key: Hashable):
        offloaded = self.offloaded_values.pop(key)
        if offloaded is not None:
            OffloadCache.keep_onloaded_values.pop(offloaded, None)

    def __contains__(self, key) -> bool:
        return key in self.offloaded_values

    def __iter__(self):
        return iter(self.offloaded_values)

    def __len__(self) -> int:
        return len(self.offloaded_values)

    @classmethod
    @contextlib.contextmanager
    def disable_offloading(cls):
        """keep every tensor onloaded after its first read until the outermost context exits"""
        if OffloadCache.offloading_disabled:
            yield
            return
        OffloadCache.offloading_disabled = True
        try:
            yield
        finally:
            OffloadCache.offloading_disabled = False
            OffloadCache.keep_onloaded_values.clear()

    @classmethod
    @contextlib.contextmanager
    def disable_onloading(cls):
        """read and assign offloaded values directly, with no device movement"""
        if OffloadCache.onloading_disabled:
            yield
            return
        OffloadCache.onloading_disabled = True
        try:
            yield
        finally:
            OffloadCache.onloading_disabled = False
