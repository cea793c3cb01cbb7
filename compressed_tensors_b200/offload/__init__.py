"""
Offloading modules to CPU, disk or another device (the reference's `compressed_tensors.offload`).

An offloaded module's `_parameters` and `_buffers` are `OffloadCache`s: assigning a tensor offloads it, reading it onloads it to the
module's onload device, and the module's forward moves its inputs there first.  `CPUCache` keeps tensors in pinned host memory and
onloads them with asynchronous copies; `DiskCache` keeps one safetensors file per tensor; `DeviceCache` keeps them on a device.

`ModelCompressor.compress_model` / `decompress_model` read CPU- and disk-offloaded modules where they are kept (under
`disable_onloading`) and run them through the host pipeline in one queue; see compressors/model_compressors/batched.py.

Not implemented, and refused by name: the distributed caches, conversion to / from accelerate, and `load_offloaded_model`.
"""
from __future__ import annotations

import contextlib
from collections.abc import Iterable
from typing import Literal

import torch

from ..utils.helpers import deprecated, patch_attr
from .cache import OffloadCache
from .convert import from_accelerate, to_accelerate
from .dispatch import dispatch_model, dispatch_with_map, get_device_map, offload_model, remove_dispatch, set_onload_device
from .load import load_offloaded_model
from .module import offload_module, remove_module_offload, unwrap_offload_forward
from .utils import as_single_threaded, get_module_device, module_size, move_module_tensor, to_meta

__all__ = [
    "set_onload_device", "offload_model", "dispatch_model", "remove_dispatch", "dispatch_with_map", "get_device_map",
    "offload_module", "remove_module_offload", "get_cache_kwargs", "get_cache_init_kwargs",
    "load_offloaded_model", "from_accelerate", "to_accelerate",
    "disable_onloading", "disable_offloading",
    "update_offload_parameter", "get_execution_device", "get_offloaded_device", "register_offload_module",
    "unwrap_offload_forward", "align_modules", "align_module_device",
    "is_distributed", "as_single_threaded", "to_meta", "module_size", "OffloadCache",
]


@contextlib.contextmanager
def disable_offloading():
    """tensors onloaded inside the context stay onloaded (later reads hit the kept copy) until the outermost context exits"""
    with OffloadCache.disable_offloading():
        yield


@contextlib.contextmanager
def disable_onloading():
    """reads return offloaded tensors as they are kept, and assignments store tensors as given: no device movement"""
    with OffloadCache.disable_onloading():
        yield


def update_offload_parameter(module: torch.nn.Module, name: str, data: torch.Tensor):
    """Write `data` into the existing parameter / buffer `name` of `module`.  For an offloaded module the offloaded value is
    updated (in place when the shape is unchanged) together with any onloaded copy kept by `disable_offloading`.  Only one caller
    may update a given tensor at a time."""
    if isinstance(module._parameters, OffloadCache):
        if name in module._parameters:
            module._parameters[name] = data
        elif name in module._buffers:
            module._buffers[name] = data
        else:
            raise AttributeError(f"{type(module)} has no attribute {name}")
        return
    if name not in module._parameters and name not in module._buffers:
        raise AttributeError(f"{type(module)} has no attribute {name}")
    with torch.no_grad():
        getattr(module, name).copy_(data)


def get_execution_device(module: torch.nn.Module, default: torch.device | None = None) -> torch.device | Literal["disk"]:
    """the device the module's inputs go to: its onload device when offloaded, else the device of its first tensor"""
    if isinstance(module._parameters, OffloadCache):
        return module._parameters.onload_device
    return get_module_device(module, default)


def get_offloaded_device(module: torch.nn.Module, default: torch.device | None = None) -> torch.device | Literal["disk"]:
    """where the module's tensors are kept between uses: its offload device when offloaded, else the device of its first tensor"""
    if isinstance(module._parameters, OffloadCache):
        return module._parameters.offload_device
    return get_module_device(module, default)


@deprecated("compressed_tensors.offload::get_cache_init_kwargs")
def get_cache_kwargs(module: torch.nn.Module, default: dict | None = None) -> dict:
    """the cache constructor arguments beyond the devices (`offload_dir` of a disk-offloaded module), added to `default`"""
    kwargs = dict(default or {})
    if isinstance(module._parameters, OffloadCache) and hasattr(module._parameters, "offload_dir"):
        kwargs["offload_dir"] = module._parameters.offload_dir
    return kwargs


def get_cache_init_kwargs(module: torch.nn.Module, default: dict | None = None) -> dict:
    """the `offload_module` arguments that offload another module like `module`: onload / offload device and `offload_dir`"""
    kwargs = dict(default or {})
    kwargs["onload_device"] = get_execution_device(module, kwargs.get("onload_device"))
    kwargs["offload_device"] = get_offloaded_device(module, kwargs.get("offload_device"))
    if hasattr(module._parameters, "offload_dir"):
        kwargs["offload_dir"] = module._parameters.offload_dir
    return kwargs


def register_offload_module(base: torch.nn.Module, name: str, module: torch.nn.Module):
    """`base.register_module(name, module)`, offloading `module` like `base` first when `base` is offloaded"""
    if isinstance(base._parameters, OffloadCache):
        offload_module(module, **get_cache_init_kwargs(base))
    base.register_module(name, module)


@contextlib.contextmanager
def align_modules(modules: torch.nn.Module | Iterable[torch.nn.Module], execution_device: torch.device | None = None):
    """`align_module_device` for several modules at once"""
    if isinstance(modules, torch.nn.Module):
        modules = (modules,)
    with contextlib.ExitStack() as stack:
        for module in modules:
            stack.enter_context(align_module_device(module, execution_device))
        yield


@contextlib.contextmanager
def align_module_device(module: torch.nn.Module, execution_device: torch.device | None = None):
    """Inside the context the module's tensors are on its execution device (or `execution_device`): an offloaded module keeps its
    onloaded tensors (offloading disabled), a plain module has its direct parameters moved there and back."""
    if isinstance(module._parameters, OffloadCache):
        assert isinstance(module._buffers, OffloadCache)
        with module._parameters.disable_offloading():
            if execution_device is None:
                yield
            else:
                with patch_attr(module._parameters, "onload_device", execution_device), \
                        patch_attr(module._buffers, "onload_device", execution_device):
                    yield
        return
    devices = {name: p.device for name, p in module.named_parameters(recurse=False)}
    for name in devices:
        move_module_tensor(module, name, execution_device)
    try:
        yield
    finally:
        for name, device in devices.items():
            move_module_tensor(module, name, device)


def is_distributed() -> bool:
    from ..distributed import is_distributed as _d

    return _d()
