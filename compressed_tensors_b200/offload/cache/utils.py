"""Error reporting shared by the caches."""
from __future__ import annotations

import errno
import logging
from functools import wraps

__all__ = ["catch_cpu_mem_error"]

_LOGGER = logging.getLogger(__name__)

_HOST_OOM_MARKERS = ("defaultcpuallocator", "can't allocate memory", "cannot allocate memory", "failed to allocate", "out of memory",
                     "mmap", "shm_open")


def _host_out_of_memory(exc: BaseException) -> bool:
    return getattr(exc, "errno", None) == errno.ENOMEM or any(m in str(exc).lower() for m in _HOST_OOM_MARKERS)


def catch_cpu_mem_error(func):
    """re-raise host out-of-memory errors of `func` after logging what to do about them (once per exception)"""

    @wraps(func)
    def wrapper(*args, **kwargs):
        try:
            return func(*args, **kwargs)
        except (RuntimeError, OSError) as exc:
            if not getattr(exc, "_ct_logged", False) and _host_out_of_memory(exc):
                _LOGGER.warning("CPU offloading ran out of host memory or mmap descriptors: offload to disk "
                                "(offload_device='disk') or raise the OS mmap limit")
                exc._ct_logged = True
            raise

    return wrapper
