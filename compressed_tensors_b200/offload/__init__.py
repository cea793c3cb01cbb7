"""
Touch points of the reference's `offload` sub-package that the hot path and its tests import (SURVEY.md Appendix C).
The offload caches themselves (CPU / disk / device caches, dispatch hooks) are control plane and out of scope: this engine keeps
modules where the caller put them, so these helpers are the "no offloading" behaviour of the reference functions
(src/compressed_tensors/offload/__init__.py:113-149 and friends) -- a plain in-place update, a no-op context, the module's device.
"""
from __future__ import annotations

import contextlib

import torch

__all__ = ["update_offload_parameter", "disable_onloading", "disable_offloading", "get_execution_device", "is_distributed"]


def update_offload_parameter(module: torch.nn.Module, name: str, data: torch.Tensor):
    """copy `data` into an existing parameter / buffer of a (non-offloaded) module"""
    if name not in module._parameters and name not in module._buffers:
        raise AttributeError(f"{type(module)} has no attribute {name}")
    with torch.no_grad():
        getattr(module, name).copy_(data)


@contextlib.contextmanager
def disable_onloading():
    """nothing is ever offloaded here, so there is nothing to disable"""
    yield


@contextlib.contextmanager
def disable_offloading():
    """nothing is ever offloaded here, so there is nothing to keep onloaded"""
    yield


def get_execution_device(module: torch.nn.Module, default: torch.device | None = None) -> torch.device:
    for t in module.parameters(recurse=False):
        return t.device
    for t in module.buffers(recurse=False):
        return t.device
    return default if default is not None else torch.device("cpu")


def is_distributed() -> bool:
    from ..distributed import is_distributed as _d

    return _d()


def _no_offload(name: str):
    def refuse(*args, **kwargs):
        raise NotImplementedError(f"compressed_tensors_b200.offload.{name}: CPU / disk offloading of modules is a separate subsystem of the "
                                  "reference (offload/dispatch.py, offload/cache/) and is not part of this engine (DESIGN.md section 7)")

    refuse.__name__ = name
    return refuse


# importable so that the reference's lifecycle test files load; calling them says what is missing instead of pretending to offload
set_onload_device = _no_offload("set_onload_device")
offload_module = _no_offload("offload_module")
offload_model = _no_offload("offload_model")
dispatch_model = _no_offload("dispatch_model")
__all__ += ["set_onload_device", "offload_module", "offload_model", "dispatch_model"]


class OffloadCache(dict):
    """the type the reference's offloaded modules use for `module._parameters` / `_buffers` (offload/cache/base.py).  Nothing here ever
    creates one: `isinstance(module._parameters, OffloadCache)` is how callers ask "is this module offloaded?", and the answer is no."""

    def __init__(self, *args, **kwargs):
        raise NotImplementedError("compressed_tensors_b200 does not offload modules (DESIGN.md section 7)")


def module_size(module: torch.nn.Module, recurse: bool = True) -> int:
    """bytes of the module's parameters and buffers (offload/utils.py:144-158); the weight of a module in greedy_bin_packing"""
    from itertools import chain

    return sum((t.nbytes for t in chain(module.parameters(recurse=recurse), module.buffers(recurse=recurse))), 0)


def to_meta(module: torch.nn.Module) -> None:
    """replace the module's direct parameters and buffers by meta tensors of the same shape / dtype (offload/utils.py:189-209): what
    the ranks that do not own a module keep while its owner compresses it"""
    from ..utils.module import get_direct_state_dict, replace_direct_state_dict

    state = get_direct_state_dict(module)
    replace_direct_state_dict(module, {k: (v.to("meta") if v is not None else None) for k, v in state.items()})


@contextlib.contextmanager
def as_single_threaded():
    """the reference swaps its distributed offload caches for the local ones inside this context (offload/utils.py:212-240); without
    offload caches there is nothing to swap"""
    yield


__all__ += ["OffloadCache", "module_size", "to_meta", "as_single_threaded"]
