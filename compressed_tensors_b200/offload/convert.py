"""Conversion between accelerate's offloading hooks and this package's offload caches: not implemented (DESIGN.md section 7)."""
from __future__ import annotations

__all__ = ["from_accelerate", "to_accelerate"]


def _refused(name: str):
    def refuse(*args, **kwargs):
        raise NotImplementedError(f"compressed_tensors_b200.offload.convert.{name}: converting to / from accelerate's offloading is not "
                                  "implemented in compressed_tensors_b200 (DESIGN.md section 7)")

    refuse.__name__ = name
    return refuse


from_accelerate = _refused("from_accelerate")
to_accelerate = _refused("to_accelerate")
