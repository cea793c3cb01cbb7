"""Offload caches: the mappings that replace an offloaded module's `_parameters` / `_buffers`."""
from .base import OffloadCache
from .cpu import CPUCache
from .device import DeviceCache
from .disk import DiskCache
from .utils import catch_cpu_mem_error

__all__ = ["OffloadCache", "CPUCache", "DeviceCache", "DiskCache", "catch_cpu_mem_error"]
