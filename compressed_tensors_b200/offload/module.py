"""Offloading one module: swap its tensor dicts for caches and wrap its forward so that inputs follow the weights."""
from __future__ import annotations

import contextlib
from functools import wraps

import torch

from .cache.base import OffloadCache
from .utils import send_tensors

__all__ = ["offload_module", "remove_module_offload", "unwrap_offload_forward"]


def offload_module(module: torch.nn.Module, onload_device: torch.device | str, offload_device: torch.device | str, **kwargs):
    """Offload the module's direct parameters and buffers to `offload_device` (a device, "cpu" or "disk"; `kwargs` go to the cache,
    e.g. `offload_dir` for disk).  Reading them onloads them to `onload_device`, and `forward` first moves its tensor arguments
    there."""
    if isinstance(module._parameters, OffloadCache):
        raise ValueError("Attempted to offload a module twice. Please call `remove_module_offload` first.")

    cache_cls = OffloadCache.cls_from_device(offload_device)
    module._parameters = cache_cls.from_mapping(module._parameters, onload_device, offload_device, **kwargs)
    module._buffers = cache_cls.from_mapping(module._buffers, onload_device, offload_device, **kwargs)

    module._original_forward_func = module.forward.__func__

    @wraps(module._original_forward_func)
    def forward(self, *args, **kwargs):
        if not OffloadCache.onloading_disabled and isinstance(self._parameters, OffloadCache):
            device = self._parameters.onload_device
            args, kwargs = send_tensors(args, device=device), send_tensors(kwargs, device=device)
        return self._original_forward_func(self, *args, **kwargs)

    module.forward = forward.__get__(module)
    return module


def remove_module_offload(module: torch.nn.Module, onload_tensors: bool = False):
    """Undo `offload_module`: plain dicts again, holding the onloaded tensors (`onload_tensors`) or the offloaded ones, and the
    original forward."""
    if not isinstance(module._parameters, OffloadCache):
        return
    params, buffers = module._parameters, module._buffers
    assert isinstance(buffers, OffloadCache)
    if onload_tensors:
        module._parameters = {k: params.onload(v) for k, v in params.offloaded_values.items()}
        module._buffers = {k: buffers.onload(v) for k, v in buffers.offloaded_values.items()}
    else:
        module._parameters = params.offloaded_values
        module._buffers = buffers.offloaded_values
    module.forward = module._original_forward_func.__get__(module)
    del module._original_forward_func


@contextlib.contextmanager
def unwrap_offload_forward(module: torch.nn.Module):
    """Inside the context the module's forward is its own, without the offload wrapper; whatever forward it has on exit is wrapped
    again.  For code that replaces `module.forward` (e.g. quantized forward) on a module that may be offloaded."""
    if not hasattr(module, "_original_forward_func"):
        yield
        return
    wrapper = module.forward
    module.forward = module._original_forward_func.__get__(module)
    try:
        yield
    finally:
        module._original_forward_func = module.forward.__func__
        module.forward = wrapper
