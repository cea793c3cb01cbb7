"""
Hadamard matrices of the transform factories (the reference's transform/utils/hadamard.py).

`random_hadamard_matrix` is diag(Q) . H_n for a power of two n with Q drawn from the generator exactly as the reference draws it:
the reference builds its matrix from a table of known Hadamard matrices whose entry for every power of two except 32 is Sylvester's
matrix, so for those orders the two are equal.  The table itself is not part of this package: the non-power-of-two orders and 32
raise NotImplementedError (DESIGN.md section 1, row (h)).
"""
from __future__ import annotations

import torch

__all__ = ["random_hadamard_matrix", "deterministic_hadamard_matrix", "is_pow2"]


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
    """diag(Q) . H with Q a vector of random signs drawn from `gen` (on the CPU, in `dtype`)"""
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
