"""
Hadamard matrices of the transform factories (the reference's transform/utils/hadamard.py).

`random_hadamard_matrix` is diag(Q) . H_n for a power of two n with Q drawn from the generator exactly as the reference draws it:
the reference builds its matrix from a table of known Hadamard matrices whose entry for every power of two except 32 is Sylvester's
matrix, so for those orders the two are equal.  The table itself is not part of this package, so on a real device the other orders
(n = K * 2^m with a table core K that is not a power of two, and 32) raise NotImplementedError (DESIGN.md section 1, row (h)).  On
the meta device every order of the table is built: the signs are drawn as the reference draws them and an empty [n, n] tensor is
returned, so a model can be built on meta and its transform weights loaded from a checkpoint, which carries the whole matrix.
"""
from __future__ import annotations

import torch

__all__ = ["random_hadamard_matrix", "deterministic_hadamard_matrix", "is_pow2", "table_core_order"]


def deterministic_hadamard_matrix(size: int, dtype: torch.dtype = torch.bfloat16, device: torch.device = torch.device("cpu")) -> torch.Tensor:
    """Sylvester's Hadamard matrix of order `size` (a power of two): H_2k = [[H_k, H_k], [H_k, -H_k]]"""
    if size <= 0:
        raise ValueError("Cannot construct deterministic hadamard of size <= 0")
    if not is_pow2(size):
        raise ValueError("Cannot construct deterministic hadamard of size != 2^n")
    H = torch.ones((1, 1), dtype=dtype, device=device)
    while H.shape[0] < size:
        H = torch.cat((torch.cat((H, H), dim=1), torch.cat((H, -H), dim=1)), dim=0)
    return H


def random_hadamard_matrix(size: int, dtype: torch.dtype = torch.bfloat16, device: torch.device = torch.device("cpu"),
                           gen: torch.Generator | None = None) -> torch.Tensor:
    """diag(Q) . H with Q a vector of random signs drawn from `gen` (on the CPU, in `dtype`); on the meta device, for every order of
    the reference's table, an empty [size, size] tensor after drawing Q"""
    if torch.device(device).type == "meta" and table_core_order(size) is not None:
        torch.randint(low=0, high=2, size=(size,), generator=gen, dtype=dtype)
        return torch.empty((size, size), dtype=dtype, device="meta")
    if not is_pow2(size) or size == 32:
        raise NotImplementedError(
            f"random-hadamard of size {size} needs a known Hadamard matrix of a non-Sylvester order, which this package does not ship; "
            "powers of two other than 32 are supported")
    Q = torch.randint(low=0, high=2, size=(size,), generator=gen, dtype=dtype)
    Q = Q.to(device=device) * 2 - 1
    return Q.unsqueeze(1) * deterministic_hadamard_matrix(size, dtype, device)


def is_pow2(n: int) -> bool:
    """True iff `n` is a power of two"""
    return n > 0 and (n & (n - 1)) == 0


def table_core_order(n: int) -> int | None:
    """the order K of the core the reference's table gives for a matrix of order n = K * 2^m: n itself up to 256, else the K in
    (128, 256]; the table holds 1, 2 and every multiple of 4 up to 256.  None when the table has no such core."""
    if n < 1:
        return None
    k = n
    while k > 256 and k % 2 == 0:
        k //= 2
    return k if k <= 256 and (k in (1, 2) or k % 4 == 0) else None
