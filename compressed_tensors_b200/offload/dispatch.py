"""Placing whole models: offload every module to where it is, dispatch across devices by memory, or follow a device map."""
from __future__ import annotations

import logging
import os
from collections.abc import Container
from typing import Any, Optional, TypeVar

import torch

from ..utils.helpers import deprecated
from .cache import OffloadCache
from .module import offload_module, remove_module_offload
from .utils import get_module_device, get_module_sizes, module_size

__all__ = ["set_onload_device", "offload_model", "dispatch_with_map", "get_device_map", "dispatch_model", "remove_dispatch",
           "get_device_memory", "DeviceMap"]

_LOGGER = logging.getLogger(__name__)

ModelType = TypeVar("ModelType", bound=torch.nn.Module)
# module name -> (onload device, offload device); an offload device of None leaves the module as it is
DeviceMap = dict[str, tuple[Optional[torch.device], Optional[torch.device | str]]]


def set_onload_device(model: ModelType, onload_device: torch.device | str) -> ModelType:
    """Make every module of `model` onload to `onload_device`.  Modules already offloaded keep their offloaded tensors; the others
    are offloaded to the device they are on now."""
    for module in model.modules():
        if isinstance(module._parameters, OffloadCache):
            module._parameters.onload_device = onload_device
            module._buffers.onload_device = onload_device
        else:
            offload_module(module, onload_device, get_module_device(module, torch.device("cpu")))
    return model


@deprecated("set_onload_device")
def offload_model(model: ModelType, onload_device: torch.device | str, offload_device: Any = None) -> ModelType:
    """deprecated: `set_onload_device`"""
    return set_onload_device(model, onload_device)


def dispatch_with_map(model: torch.nn.Module, device_map: DeviceMap, offload_dir: Optional[str] = None, show_progress: bool = True):
    """Offload each module named in `device_map` to its (onload, offload) pair; `offload_dir` is where disk offloads go.  Names
    that do not exist in this model (e.g. experts another rank holds) are skipped."""
    import tqdm

    for name, (onload, offload) in tqdm.tqdm(list(device_map.items()), desc="Dispatching model", disable=not show_progress):
        try:
            module = model.get_submodule(name)
        except AttributeError:
            _LOGGER.debug("Skipping '%s' from device map: not present locally", name)
            continue
        if offload == "disk":
            offload_module(module, onload, offload, offload_dir=offload_dir)
        elif offload is not None:
            offload_module(module, onload, offload)


def get_device_map(model: torch.nn.Module, default_device: torch.device = torch.device("cpu")) -> DeviceMap:
    """the (onload, offload) devices of every module of `model`; `default_device` for modules without tensors"""
    from . import get_execution_device, get_offloaded_device

    return {name: (get_execution_device(m, default_device), get_offloaded_device(m, default_device))
            for name, m in model.named_modules(remove_duplicate=False)}


def _greedy(sizes, memory: dict, reserve: float):
    """place modules in order, each on the first device (in `memory` order, never going back) with room for it plus `reserve`;
    returns the placements made before running out of devices and the memory left"""
    left = dict(memory)
    devices = list(left)
    placed, d = [], 0
    for module, size in sizes:
        while d < len(devices) and size > left[devices[d]] - reserve:
            d += 1
        if d == len(devices):
            break
        placed.append((module, devices[d], devices[d]))
        left[devices[d]] -= size
    return placed, left


def dispatch_model(model: ModelType, device_memory: dict[torch.device, int] | None = None, extra_memory: int | None = None,
                   no_split_modules: Container[str] | None = None) -> ModelType:
    """Spread `model` over the devices for generation: modules stay whole (those in `no_split_modules`, default the model's
    `_no_split_modules`, and every module with direct tensors), are placed in `model.modules()` order, and are kept on their
    device.  The placement keeps as much memory free on every device as possible, at least `extra_memory` (default: 5% of the
    model, at least 1 GB, plus one 2048-token activation of a transformers model).  When the model does not fit, the tail of it is
    offloaded to CPU and onloaded to the last device.  Existing offloads are removed first."""
    if no_split_modules is None:
        no_split_modules = getattr(model, "_no_split_modules", None) or ()
    if device_memory is None:
        device_memory = get_device_memory()
    if len(device_memory) == 0:
        raise MemoryError("Did not find any devices to dispatch model to")
    sizes = get_module_sizes(model, no_split_modules)
    if len(sizes) == 0:
        raise ValueError("Model does not have any modules")

    if extra_memory is None:
        extra_memory = max(module_size(model) * 0.05, 1e9)
        try:
            from transformers import PreTrainedModel
        except ImportError:
            PreTrainedModel = ()
        if PreTrainedModel and isinstance(model, PreTrainedModel):
            dtype = getattr(model, "dtype", torch.bfloat16)
            extra_memory += 2048 * getattr(getattr(model, "config", None), "intermediate_size", 256) * dtype.itemsize

    placed, left = _greedy(sizes, device_memory, extra_memory)
    if len(placed) == len(sizes):
        # the largest reserve that still places everything (bisection over whole bytes)
        lo, hi = int(extra_memory), int(min(device_memory.values()))
        while lo < hi:
            mid = (lo + hi + 1) // 2
            if len(_greedy(sizes, device_memory, mid)[0]) == len(sizes):
                lo = mid
            else:
                hi = mid - 1
        extra_memory = lo
        placed, _ = _greedy(sizes, device_memory, extra_memory)
    else:
        size_of = dict((id(m), s) for m, s in sizes)
        last = placed[-1][1] if placed else next(iter(device_memory))
        largest = max(s for _, s in sizes[len(placed):])
        # take modules back off the last device until the largest CPU-offloaded module can be onloaded there
        while largest + extra_memory > left[last]:
            if not placed:
                raise ValueError(f"Cannot fit no_split module of size {largest} bytes into any device: {device_memory}")
            module, last, _ = placed.pop()
            left[last] += size_of[id(module)]
            largest = max(largest, size_of[id(module)])
        placed += [(module, last, "cpu") for module, _ in sizes[len(placed):]]
        _LOGGER.warning("Forced to offload modules due to insufficient gpu resources")

    plan = {sub: (onload, offload) for module, onload, offload in placed for sub in module.modules()}
    for module in model.modules():
        remove_module_offload(module, onload_tensors=True)
        if module in plan:
            offload_module(module, *plan[module])
    _LOGGER.debug("Dispatched model with %s bytes of extra memory", extra_memory)
    return model


def get_device_memory() -> dict[torch.device, int]:
    """total memory of every CUDA device (only the current one under torch.distributed); system RAM as "cpu" without CUDA"""
    if not torch.cuda.is_available():
        return {torch.device("cpu"): os.sysconf("SC_PAGE_SIZE") * os.sysconf("SC_PHYS_PAGES")}
    import torch.distributed as dist

    if dist.is_available() and dist.is_initialized():
        idx = torch.cuda.current_device()
        return {torch.device("cuda"): torch.cuda.mem_get_info(idx)[1]}
    return {torch.device("cuda", i): torch.cuda.mem_get_info(i)[1] for i in range(torch.cuda.device_count())}


def remove_dispatch(module: torch.nn.Module, onload_tensors: bool = False) -> torch.nn.Module:
    """remove the offloading of `module` and all its submodules"""
    for sub in module.modules():
        remove_module_offload(sub, onload_tensors)
    return module
