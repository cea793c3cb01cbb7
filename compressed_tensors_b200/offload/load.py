"""Loading a checkpoint straight into an offloaded model: not implemented (DESIGN.md section 7)."""
from __future__ import annotations

__all__ = ["load_offloaded_model"]


def load_offloaded_model(*args, **kwargs):
    raise NotImplementedError("compressed_tensors_b200.offload.load_offloaded_model: loading a checkpoint into an offloaded model is not "
                              "implemented in compressed_tensors_b200 (DESIGN.md section 7); load the model, then call "
                              "`set_onload_device`, `dispatch_model` or `dispatch_with_map`")
