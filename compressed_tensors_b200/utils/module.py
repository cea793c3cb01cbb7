"""
Direct (non-recursive) state-dict access used by compress_module / decompress_module
(mirror of utils/module.py:13-65).
"""
from __future__ import annotations

from itertools import chain

import torch

__all__ = ["get_direct_state_dict", "replace_direct_state_dict"]


def get_direct_state_dict(module: torch.nn.Module) -> dict[str, torch.Tensor]:
    """parameters and buffers of this module only, as plain tensors"""
    out = {}
    for name, t in chain(module._parameters.items(), module._buffers.items()):
        out[name] = t.data if isinstance(t, (torch.nn.Parameter, torch.nn.Buffer)) else t
    return out


def replace_direct_state_dict(module: torch.nn.Module, new_state_dict: dict[str, torch.Tensor]):
    """drop names that disappeared, (re)register everything else as frozen Parameters (utils/module.py:34-65).

    On an offloaded module the writes go through its caches: a new value is offloaded (pinned host memory, a new file), a value
    that is the offloaded tensor itself, or a view of exactly its bytes, is left where it is -- a buffer passed through unchanged
    stays a buffer, where the reference re-registers it as a parameter.

    Works on the module's `_parameters` / `_buffers` dicts directly: `delattr` / `setattr` go through nn.Module's attribute
    machinery (type checks, hook lookups, three dict probes per call), which made this function the largest share of the per-module
    host time of a whole-model compress -- at 8 ranks every rank re-registers ~1500 tensors of the modules it only mirrors on meta."""
    from ..offload.cache import OffloadCache

    params, bufs = module._parameters, module._buffers
    if isinstance(params, OffloadCache):
        _replace_offloaded(params, bufs, new_state_dict)
        return
    for name in [n for n in chain(params, bufs) if n not in new_state_dict]:
        params.pop(name, None)
        bufs.pop(name, None)
    for name, value in new_state_dict.items():
        bufs.pop(name, None)
        module.__dict__.pop(name, None)
        params[name] = torch.nn.Parameter(value, requires_grad=False) if value is not None else None


def _same_bytes(a: torch.Tensor, b: torch.Tensor) -> bool:
    return a is b or (a.device.type != "meta" and a.device == b.device and a.dtype == b.dtype and a.shape == b.shape
                      and a.stride() == b.stride() and a.data_ptr() == b.data_ptr())


def _replace_offloaded(params, bufs, new_state_dict: dict[str, torch.Tensor]):
    old = {**bufs.offloaded_values, **params.offloaded_values}
    for name in [n for n in old if n not in new_state_dict]:
        del (params if name in params else bufs)[name]
    for name, value in new_state_dict.items():
        if name in old:
            if old[name] is value or (old[name] is not None and value is not None and _same_bytes(old[name], value)):
                continue   # unchanged: stays where it is kept (a buffer stays a buffer, a DiskCache file stays its file)
            del (params if name in params else bufs)[name]
        params[name] = torch.nn.Parameter(value, requires_grad=False) if value is not None else None
