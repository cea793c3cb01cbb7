"""
`DiskCache`: every offloaded tensor is one safetensors file under `offload_dir`, and the cache keeps a meta tensor of the same
shape / dtype in its place.  The class-wide `index` maps each meta tensor to its file, the tensor name inside it, and its dtype.

Only files this class created (their names start with `ct_disk_cache`) are ever rewritten or deleted; an index entry may point at
another file (a symlink into a checkpoint), which is replaced by a new file on the first update.
"""
from __future__ import annotations

import os
from pathlib import Path
from typing import Literal, Optional

import torch

from ..utils import send_tensors, to_tensor
from .base import OffloadCache

__all__ = ["DiskCache"]


def _rank() -> int:
    import torch.distributed as dist

    return dist.get_rank() if dist.is_available() and dist.is_initialized() else 0


def _safe_open_device(device) -> str:
    """`safe_open` takes a device string; an accelerator without an index means the current one"""
    device = torch.device(device)
    if device.type == "cuda":
        return f"cuda:{device.index if device.index is not None else torch.cuda.current_device()}"
    return device.type if device.index is None else str(device)


class DiskCache(OffloadCache):
    offload_device = "disk"

    # meta tensor -> {"safetensors_file", "weight_name", "dtype"} (shared by every DiskCache)
    index: dict[torch.Tensor, dict[str, str]] = dict()

    offload_dir: Path
    _ct_file_prefix = "ct_disk_cache"

    def __init__(self, onload_device: torch.device | str, offload_device: Optional[str] = None, offload_dir: Optional[str] = None):
        super().__init__(onload_device, offload_device=offload_device)
        if offload_dir is None:
            raise ValueError("Must provide an `offload_dir` to perform disk offloading (add `offload_folder` argument to `from_pretrained`)")
        self.offload_dir = Path(offload_dir).resolve()

    def read(self, offloaded: torch.Tensor | None, device="cpu") -> torch.Tensor | None:
        """the file's tensor on `device` (through `safe_open`), with the class and attributes of the offloaded tensor"""
        if offloaded is None:
            return None
        from safetensors import safe_open

        info = self.index[offloaded]
        with safe_open(info["safetensors_file"], framework="pt", device=_safe_open_device(device)) as f:
            tensor = f.get_tensor(info["weight_name"])
        return to_tensor(tensor, offloaded).to(getattr(torch, info["dtype"]))

    def onload(self, offloaded: torch.Tensor | None) -> torch.Tensor | None:
        return self.read(offloaded, self.onload_device)

    def offload(self, tensor: torch.Tensor | None, offloaded: Optional[torch.Tensor] = None) -> torch.Tensor | None:
        """write `tensor` to a new file of this cache; returns the meta tensor that stands for it"""
        if tensor is None:
            return None
        if tensor.device.type == "meta":
            assert tensor in self.index, "a meta tensor can only be offloaded to disk if it already stands for a file"
            return tensor
        from safetensors.torch import save_file

        if offloaded is None:
            offloaded = send_tensors(tensor, device="meta")
        path = self._file_for(self.offload_dir, offloaded)
        DiskCache.index[offloaded] = {"safetensors_file": path, "weight_name": "weight", "dtype": str(tensor.dtype).removeprefix("torch.")}
        save_file({"weight": tensor.detach().contiguous()}, path)
        return offloaded

    def update_offload(self, offloaded: torch.Tensor, data: torch.Tensor | None):
        if data is None:
            return
        from safetensors.torch import save_file

        assert offloaded in self.index, "Cannot find offload to update"
        info = self.index[offloaded]
        path = info["safetensors_file"]
        assert self._owns(path), f"Attempted to write to {path}"
        if os.path.islink(path):
            os.unlink(path)   # a link into a checkpoint: the update goes to a file of our own
        save_file({info["weight_name"]: data.detach().reshape_as(offloaded).to(dtype=getattr(torch, info["dtype"])).contiguous()}, path)

    def __delitem__(self, key):
        offloaded = self.offloaded_values[key]
        if not OffloadCache.onloading_disabled and offloaded is not None:
            path = self.index[offloaded]["safetensors_file"]
            if self._owns(path) and os.path.lexists(path):
                os.remove(path)
            del DiskCache.index[offloaded]
        super().__delitem__(key)

    @classmethod
    def create_checkpoint_symlink(cls, offloaded: torch.Tensor, weight_info: dict, offload_dir: str | os.PathLike | None) -> None:
        """make `offloaded` stand for a tensor of an existing checkpoint file, through a symlink in `offload_dir`"""
        if offload_dir is None:
            raise ValueError("Must provide an `offload_dir` to perform disk offloading (add `offload_folder` argument to `from_pretrained`)")
        path = cls._file_for(offload_dir, offloaded)
        os.symlink(Path(weight_info["safetensors_file"]).resolve(), path)
        cls.index[offloaded] = {"safetensors_file": path, "weight_name": weight_info["weight_name"], "dtype": weight_info["dtype"]}

    @classmethod
    def _owns(cls, path) -> bool:
        return os.path.basename(path).startswith(cls._ct_file_prefix)

    @classmethod
    def _file_for(cls, offload_dir, offloaded: torch.Tensor) -> str:
        return os.path.join(offload_dir, f"{cls._ct_file_prefix}_{_rank()}_{id(offloaded)}.safetensors")
