"""
`CPUCache`: offloaded tensors live in page-locked host memory, so that onloading them is an asynchronous DMA.

  * offload: a CPU tensor that is already pinned is kept as it is; anything else is copied into a new pinned tensor, which keeps
    the tensor's class, attributes and `requires_grad`.  This differs from the reference, which keeps a pageable CPU tensor
    as the same object.  So that tied weights stay tied (e.g. `embed_tokens.weight is lm_head.weight`), every cache offloading
    the same source tensor while it is alive gets the same pinned copy, and an update through one module reaches the other.
    When pinning is not possible (no CUDA device, or the pinned pool is exhausted) the tensor goes to pageable memory like
    `Tensor.to("cpu")`, and that is logged once.
  * onload: `Tensor.to(onload_device, non_blocking=True)`, ordered on the current stream; the host does not wait for it.  The copy
    records a CUDA event on that stream, kept class-wide per pinned storage (one pinned tensor can sit in several caches).  Before
    `update_offload` overwrites the pinned source, and before `__delitem__` lets it go, the host waits on that event, so no copy
    still in flight reads rewritten bytes.
"""
from __future__ import annotations

import logging
import weakref

import torch

from .base import OffloadCache
from .utils import catch_cpu_mem_error

__all__ = ["CPUCache"]

_LOGGER = logging.getLogger(__name__)


# id(source tensor) -> (weak reference to the source, its pinned copy); an entry lives as long as its source
_PINNED_COPIES: dict[int, tuple[weakref.ref, torch.Tensor]] = {}

# untyped storage pointer of a pinned tensor -> CUDA event recorded after its latest onload copy
_COPIES: dict[int, torch.cuda.Event] = {}


def _pinned(tensor: torch.Tensor) -> torch.Tensor | None:
    """a pinned host copy of `tensor` (the tensor itself if it already is one, the earlier copy if this tensor was pinned before
    and is still alive), or None when memory cannot be pinned"""
    if tensor.device.type == "cpu" and tensor.is_pinned():
        return tensor
    if tensor.device.type == "meta" or not torch.cuda.is_available():
        return None
    known = _PINNED_COPIES.get(id(tensor))
    if known is not None and known[0]() is tensor:
        return known[1]
    try:
        with torch.no_grad():
            if tensor.device.type == "cpu":
                out = tensor.pin_memory()
            else:
                out = torch.empty(tensor.shape, dtype=tensor.dtype, pin_memory=True)
                out.copy_(tensor)
    except RuntimeError:
        return None
    out.__class__ = tensor.__class__
    out.__dict__ = tensor.__dict__.copy()
    if tensor.requires_grad:
        out.requires_grad_(True)
    key = id(tensor)
    _PINNED_COPIES[key] = (weakref.ref(tensor), out)
    weakref.finalize(tensor, _PINNED_COPIES.pop, key, None)
    return out


def _storage_key(t: torch.Tensor) -> int:
    return t.untyped_storage().data_ptr()


class CPUCache(OffloadCache):
    offload_device = torch.device("cpu")

    # True once a failure to pin has been logged
    _pageable_logged = False

    def __init__(self, onload_device: torch.device | str, offload_device=None):
        super().__init__(onload_device, offload_device=offload_device)

    def onload(self, offloaded: torch.Tensor | None) -> torch.Tensor | None:
        if offloaded is None:
            return None
        device = torch.device(self.onload_device)
        with torch.no_grad():
            onloaded = offloaded.to(device, non_blocking=True)
        if onloaded is offloaded:
            return offloaded
        if device.type == "cuda" and offloaded.is_pinned():
            event = torch.cuda.Event()
            event.record(torch.cuda.current_stream(device))
            if len(_COPIES) >= 4096:   # forget copies that have finished
                for k in [k for k, e in _COPIES.items() if e.query()]:
                    del _COPIES[k]
            _COPIES[_storage_key(offloaded)] = event
        onloaded.__class__ = offloaded.__class__
        onloaded.__dict__ = offloaded.__dict__.copy()
        return onloaded

    @catch_cpu_mem_error
    def offload(self, tensor: torch.Tensor | None) -> torch.Tensor | None:
        if tensor is None:
            return None
        pinned = _pinned(tensor)
        if pinned is None:
            if tensor.device.type != "meta" and torch.cuda.is_available() and not CPUCache._pageable_logged:
                CPUCache._pageable_logged = True
                _LOGGER.warning("CPUCache: could not pin host memory for an offloaded tensor; offloaded tensors that cannot be pinned "
                                "are kept in pageable memory and onload synchronously")
            with torch.no_grad():
                pinned = tensor.to("cpu")
            if pinned is not tensor:
                pinned.__class__ = tensor.__class__
                pinned.__dict__ = tensor.__dict__.copy()
        return pinned

    @staticmethod
    def _wait_for_copies(offloaded: torch.Tensor):
        if offloaded.device.type != "cpu":
            return
        event = _COPIES.pop(_storage_key(offloaded), None)
        if event is not None:
            event.synchronize()

    @torch.no_grad()
    def update_offload(self, offloaded: torch.Tensor, data: torch.Tensor | None):
        if data is None:
            return
        self._wait_for_copies(offloaded)
        offloaded.copy_(data)

    def __delitem__(self, key):
        offloaded = self.offloaded_values.get(key, None)
        if offloaded is not None:
            self._wait_for_copies(offloaded)
        super().__delitem__(key)
