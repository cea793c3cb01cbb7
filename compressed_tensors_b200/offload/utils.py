"""
Tensor and module helpers of the offload package: moving nested tensors, module devices and sizes, and the meta / single-threaded
helpers the module-parallel compressor uses.
"""
from __future__ import annotations

import contextlib
import logging
from collections.abc import Container
from dataclasses import fields, is_dataclass
from itertools import chain
from typing import TypeVar

import torch

__all__ = ["send_tensors", "get_module_device", "move_module_tensor", "get_module_sizes", "module_size", "to_empty", "to_tensor",
           "to_meta", "as_single_threaded"]

_LOGGER = logging.getLogger(__name__)

T = TypeVar("T")
TensorT = TypeVar("TensorT", bound=torch.Tensor)


def send_tensors(value: T, *args, **kwargs) -> T:
    """`Tensor.to(*args, **kwargs)` applied to every tensor inside `value` (tensors, lists, tuples, dicts, dataclasses).  A moved
    tensor keeps its class (e.g. Parameter) and attributes; a tensor that `to` leaves where it is comes back as the same object."""
    if isinstance(value, torch.Tensor):
        with torch.no_grad():
            moved = value.to(*args, **kwargs)
        if moved is value or (moved.device == value.device and moved.data_ptr() == value.data_ptr()):
            return value
        moved.__class__ = value.__class__
        moved.__dict__ = value.__dict__.copy()
        return moved
    if isinstance(value, list):
        return [send_tensors(v, *args, **kwargs) for v in value]
    if isinstance(value, tuple):
        return tuple(send_tensors(v, *args, **kwargs) for v in value)
    if isinstance(value, dict):
        return {k: send_tensors(v, *args, **kwargs) for k, v in value.items()}
    if is_dataclass(value) and not isinstance(value, type):
        return type(value)(**{f.name: send_tensors(getattr(value, f.name), *args, **kwargs) for f in fields(value)})
    return value


def get_module_device(module: torch.nn.Module, default: torch.device | None = None) -> torch.device:
    """device of the module's first parameter (else buffer), searched recursively; `default` (else CPU) when it has none"""
    tensor = next(module.parameters(), None)
    if tensor is None:
        tensor = next(module.buffers(), None)
    if tensor is not None:
        return tensor.device
    if default is not None:
        return default
    _LOGGER.warning("Unable to get the execution device of %s, falling back to CPU", type(module).__name__)
    return torch.device("cpu")


def move_module_tensor(module: torch.nn.Module, name: str, device: int | str | torch.device):
    """move one direct parameter or buffer of `module` to `device`"""
    if name in module._parameters:
        module._parameters[name] = send_tensors(module._parameters[name], device=device)
    elif name in module._buffers:
        module._buffers[name] = send_tensors(module._buffers[name], device=device)


def get_module_sizes(model: torch.nn.Module, no_split_modules: Container[str] = tuple()) -> list[tuple[torch.nn.Module, int]]:
    """the modules that must stay whole, in `model.modules()` order, with their sizes in bytes.  A module stays whole when its
    class name is in `no_split_modules` or when it has direct tensors (so that its children cannot land on another device)."""
    sizes = []

    def visit(module: torch.nn.Module):
        whole = type(module).__name__ in no_split_modules or module_size(module, recurse=False) > 0
        size = module_size(module, recurse=whole)
        if size > 0:
            sizes.append((module, size))
        if not whole:
            for child in module.children():
                visit(child)

    visit(model)
    return sizes


def module_size(module: torch.nn.Module, recurse: bool = True) -> int:
    """bytes of the module's parameters and buffers, read where they are kept (offloaded modules are not onloaded)"""
    from . import disable_onloading

    with disable_onloading():
        return sum((t.nbytes for t in chain(module.parameters(recurse=recurse), module.buffers(recurse=recurse))), 0)


def to_empty(tensor: TensorT, **kwargs) -> TensorT:
    """an uninitialised tensor like `tensor`, with its class and attributes"""
    empty = torch.empty_like(tensor.data, **kwargs)
    empty.__class__ = tensor.__class__
    empty.__dict__ = tensor.__dict__.copy()
    return empty


def to_tensor(dst: torch.Tensor, src: TensorT) -> TensorT:
    """give `dst` the class, attributes and requires_grad of `src`"""
    dst.__class__ = src.__class__
    dst.__dict__ = src.__dict__.copy()
    dst.requires_grad = src.requires_grad
    return dst


def to_meta(module: torch.nn.Module) -> None:
    """replace the module's direct parameters and buffers by meta tensors of the same shape / dtype: what the ranks that do not
    own a module keep while its owner compresses it.  An offloaded module's offloaded values are replaced, not onloaded."""
    from ..utils.module import get_direct_state_dict, replace_direct_state_dict
    from . import disable_onloading

    with disable_onloading():
        state = get_direct_state_dict(module)
        replace_direct_state_dict(module, {k: send_tensors(v, device="meta") for k, v in state.items()})


@contextlib.contextmanager
def as_single_threaded():
    """the reference swaps its distributed offload caches for the local ones inside this context; the distributed caches are
    not implemented here, so every cache already is the local one"""
    yield
