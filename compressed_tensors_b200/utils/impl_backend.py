"""
Op-level backend hook, same surface and semantics as the reference's ImplBackend (utils/impl_backend.py:23-134):

    @ImplBackend.register(name, req, priority)   a backend of op `name`; tried in priority order when `req(*args, **kwargs)` is true;
                                                 priority "disable" skips registration
    @ImplBackend.entrypoint(name)                the decorated body is the EAGER implementation: it runs when no backend accepts the
                                                 arguments, and always when CT_ENFORCE_EAGER is set (impl_backend.py:14-20, :98-123)
    ImplBackend.call(fn_name, ...)               call one registered function by its __name__, bypassing the checks (tests)

In this engine the sm_90a kernels are the backend (registered by ops.py for the seven per-tensor hot-path ops and hadamard_transform with
req = "a CUDA device is usable") and the eager body is the library's OWN host code, the `device = -1` twins of the C ABI
(csrc/cpu_twin.cu) -- not torch eager.  The reference reads CT_ENFORCE_EAGER once at import; here it is read at call time so that
a test can flip it.
"""
from __future__ import annotations

import functools
import os
from typing import Callable

__all__ = ["ImplBackend", "enforce_eager"]


def enforce_eager() -> bool:
    return os.environ.get("CT_ENFORCE_EAGER", "") not in ("", "0", "false", "False")


class ImplBackend:
    _backends: dict[str, list[tuple[Callable, Callable, int]]] = {}
    _fn_registry: dict[str, Callable] = {}    # fn.__name__ -> function (backends and eager bodies)

    @classmethod
    def register(cls, name: str, req: Callable[..., bool] = lambda *a, **k: True, priority="0"):
        def decorator(backend_fn: Callable) -> Callable:
            if priority == "disable":
                return backend_fn
            cls._add_to_registry(backend_fn)
            cls._backends.setdefault(name, []).append((backend_fn, req, int(priority)))
            cls._backends[name].sort(key=lambda entry: entry[2])
            return backend_fn

        return decorator

    @classmethod
    def call(cls, fn_name: str, *args, **kwargs):
        if fn_name not in cls._fn_registry:
            raise KeyError(f"No registered backend named '{fn_name}'. Available: {list(cls._fn_registry)}")
        return cls._fn_registry[fn_name](*args, **kwargs)

    @classmethod
    def entrypoint(cls, name: str) -> Callable:
        def decorator(fallback_fn: Callable) -> Callable:
            cls._add_to_registry(fallback_fn)

            @functools.wraps(fallback_fn)
            def wrapper(*args, **kwargs):
                if not enforce_eager():
                    for backend_fn, req, _ in cls._backends.get(name, []):
                        if req(*args, **kwargs):
                            return backend_fn(*args, **kwargs)
                return fallback_fn(*args, **kwargs)

            return wrapper

        return decorator

    @classmethod
    def _add_to_registry(cls, fn: Callable):
        fn_name = fn.__name__
        if fn_name in cls._fn_registry:
            raise ValueError(f"A backend with function name '{fn_name}' is already registered. Backend function names must be unique across all ops.")
        cls._fn_registry[fn_name] = fn
