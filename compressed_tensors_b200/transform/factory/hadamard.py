"""
The `hadamard` factory (the reference's transform/factory/hadamard.py).

A HadamardTransform holds the dense matrix (`weight`, n x n, in the scheme's precision, float64 for the weight locations) and, with
`randomize`, the permutation `perm`, exactly as the reference does, so state dicts and checkpoints are the same.  Its forward runs
the Walsh-Hadamard kernel (`ops.hadamard_transform`) when `weight` is verified to be diag(Q) . H with H Sylvester's matrix (Q is
read from the first column; the whole matrix is checked once per parameter version, and Q and perm are kept on the device of use).
Otherwise, for an order n = K * 2^m of the reference's table (K as the reference chooses it), it tries the reference's
random-hadamard structure diag(s) . (C ⊗ H_{2^m})^T with a K x K +-1 core C, read off the weight and passed to the kernel as `core`;
a trained weight (`requires_grad`), any other matrix, another precision, or an input that needs autograd runs the reference's dense
formula.
"""
from __future__ import annotations

import torch
from torch import Tensor, device, dtype
from torch.nn import Module, Parameter

from ... import ops
from ...offload import get_execution_device
from ...utils.helpers import ParameterizedDefaultDict
from .. import TransformArgs, TransformLocation, TransformScheme
from ..utils.hadamard import deterministic_hadamard_matrix, is_pow2, table_core_order
from ..utils.matrix import apply_transform_weight, get_transform_size
from .base import TransformBase, TransformFactory

__all__ = ["HadamardFactory", "HadamardTransform"]


@TransformFactory.register("hadamard")
class HadamardFactory(TransformFactory):
    """
    Factory of Hadamard transforms

    :param name: name of the scheme's group
    :param scheme: how the transforms are created and where they apply
    :param seed: seed of the generator that permutations (and random signs) are drawn from
    """

    def __init__(self, name: str, scheme: TransformScheme, seed: int | None = None):
        super().__init__(name, scheme, seed)
        self.weights = ParameterizedDefaultDict(self._create_weight)
        self.perms = ParameterizedDefaultDict(self._create_permutation)

    def create_transform(self, module: Module, args: TransformArgs):
        """a HadamardTransform for `module`; transforms of the same size, precision and device share their weight"""
        size = get_transform_size(module, args.location, self.scheme.head_dim)
        exec_device = get_execution_device(module)
        precision = self.scheme.precision if args.is_online() else torch.float64
        factory_kwargs = {"device": exec_device, "construct_device": exec_device, "precision": precision}
        weight = self.weights.get(size, factory_kwargs=factory_kwargs)
        perm = self.perms[weight] if self.scheme.randomize else None
        return HadamardTransform(weight, perm, self.scheme, args, type(module))

    def _create_weight(self, size: int, device: device, construct_device: device, precision: dtype) -> Parameter:
        data = deterministic_hadamard_matrix(size, precision, construct_device).to(device=device)
        return Parameter(data, requires_grad=self.scheme.requires_grad)

    def _create_permutation(self, weight: Parameter) -> Parameter:
        return Parameter(torch.randperm(weight.size(0), generator=self.generator), requires_grad=False)


class HadamardTransform(TransformBase):
    """
    y = value . M / sqrt(n) with M = weight, or weight[perm][:, perm], transposed with `inverse`.

    The kernel runs with copies of the signs Q and of `perm` made when they were verified.  Tracked writes (`copy_` and other
    in-place ops, `load_state_dict`, `update_offload_parameter`, assigning `weight.data = t`) change the tensor's version or storage
    and are seen on the next call.  In-place writes through `.data` (`weight.data.mul_(-1)`) are not: torch does not track them, and
    re-verifying on every call would cost a host synchronisation per call.  After such a write the kernel path keeps computing with
    the verified copies, while the dense path (an input that needs autograd, a trained weight, or a weight location the kernel does
    not take) reads the live `weight` and `perm`, so the two paths can disagree until the next tracked write.
    """

    _dynamic_tied_weights_keys: list[str] = ["weight", "perm"]

    def __init__(self, weight: Parameter, perm: Parameter | None, scheme: TransformScheme, args: TransformArgs,
                 module_type: type[torch.nn.Module]):
        super().__init__()
        self.weight = weight
        self.perm = perm
        self.scheme = scheme
        self.args = args
        self.module_type = module_type
        self._scale = torch.tensor(weight.size(0), dtype=torch.float64).sqrt()

    def forward(self, value: Tensor) -> Tensor:
        structured = _structured_signs(self.weight, self.perm, value)
        if structured is not None:
            return self._kernel(value, *structured)
        return self._dense(value)

    def _dense(self, value: Tensor) -> Tensor:
        """the reference's formula: dense product in the weight's precision, division by sqrt(n), cast back"""
        weight = self.weight
        if self.perm is not None:
            weight = weight[self.perm][:, self.perm]
        if self.args.inverse:
            weight = weight.T
        out = apply_transform_weight(weight.to(device=value.device), value.to(dtype=weight.dtype), self.args.location, self.module_type)
        return (out / self._scale).to(value.dtype)

    def _kernel(self, value: Tensor, sign: Tensor | None, perm: Tensor | None, core: Tensor | None = None) -> Tensor:
        """the same product as _dense through the butterfly: rows of `value` (or of value^T) times M or M^T"""
        n, inverse, location = self.weight.size(0), bool(self.args.inverse), TransformLocation(self.args.location)
        columns = False
        if not location.is_online():
            if self.module_type == torch.nn.Linear and location == TransformLocation.WEIGHT_INPUT:
                inverse = not inverse                      # value @ M^T
            elif self.module_type == torch.nn.Linear and location == TransformLocation.WEIGHT_OUTPUT:
                columns = True                             # M^T @ value = (value^T @ M)^T
            elif self.module_type == torch.nn.Embedding and location == TransformLocation.WEIGHT_INPUT:
                columns, inverse = True, not inverse       # M @ value = (value^T @ M^T)^T
            elif self.module_type != torch.nn.Embedding:
                return self._dense(value)                  # the reference's NotImplementedError
        x = value.T if columns else value
        if x.ndim == 0 or x.shape[-1] % n:
            return self._dense(value)
        y = ops.hadamard_transform(x, n, sign, perm, inverse, self.weight.dtype, core=core)
        return y.T if columns else y


def _structured_signs(weight: Tensor, perm: Tensor | None, value: Tensor):
    """(sign, perm, core) on value's device when the kernel computes exactly the product the dense formula asks for, else None"""
    if (weight.requires_grad or weight.device.type == "meta" or value.device.type == "meta" or weight.dtype not in (torch.float32, torch.float64)
            or value.dtype not in (torch.float32, torch.float16, torch.bfloat16) or (torch.is_grad_enabled() and value.requires_grad)):
        return None
    n = weight.size(0)
    if n > ops.HADAMARD_MAX_ORDER:
        raise NotImplementedError(f"Hadamard transforms of order {n} > {ops.HADAMARD_MAX_ORDER} are not supported")
    if n < 2 or weight.ndim != 2 or weight.size(1) != n:
        return None
    core = None
    entry = _verified(weight, "_ct_hadamard_signs", _sign_vector) if is_pow2(n) else None
    if entry is not None:
        sign = _on(entry, value.device)
    else:
        entry = _verified(weight, "_ct_hadamard_core", _core_factors) if table_core_order(n) is not None else None
        if entry is None:
            return None
        sign, core = _on(entry, value.device)
    if perm is None:
        return sign, None, core
    pentry = _verified(perm, "_ct_hadamard_perm", lambda p: p.clone() if p.ndim == 1 and p.numel() == n and _is_permutation(p) else None)
    if pentry is None:
        return None
    return sign, _on(pentry, value.device), core


def _verified(t: Tensor, attr: str, check):
    """check(t) once per version of `t`, kept on the tensor: (version, data_ptr, result on its own device, {device: copy}).

    `check` returns a snapshot that shares no memory with `t` (or True / None), and the kernel only ever receives that snapshot or
    copies of it.  A write through `t.data` bumps neither key, so it is not seen until the next tracked write; until then the
    transform keeps computing with the signs and permutation it verified, never with unverified indices."""
    cached = getattr(t, attr, None)
    if cached is None or cached[0] != t._version or cached[1] != t.data_ptr():
        with torch.no_grad():
            result = check(t.detach())
        cached = (t._version, t.data_ptr(), result, {})
        setattr(t, attr, cached)
    return None if cached[2] is None else cached


def _on(entry, dev: torch.device):
    result, copies = entry[2], entry[3]
    if result is True:          # Sylvester's matrix itself: no signs
        return None
    if dev not in copies:
        copies[dev] = tuple(t.to(dev) for t in result) if isinstance(result, tuple) else result.to(dev)
    return copies[dev]


def _sign_vector(w: Tensor):
    """True when w is H, the int8 signs Q when w is diag(Q) . H with some Q < 0, else None; checked in row blocks"""
    n = w.size(0)
    q = w[:, 0]
    if not bool(((q == 1) | (q == -1)).all()):
        return None
    cols = torch.arange(n, device=w.device)
    block = max(1, (1 << 22) // n)
    for r0 in range(0, n, block):
        rows = torch.arange(r0, min(n, r0 + block), device=w.device)
        p = rows[:, None] & cols[None, :]
        for s in (8, 4, 2, 1):
            p = p ^ (p >> s)
        expected = (1 - 2 * (p & 1)).to(w.dtype) * q[r0:r0 + block, None]
        if not torch.equal(w[r0:r0 + block], expected):
            return None
    return True if bool((q == 1).all()) else q.to(torch.int8).contiguous()   # w is fp32 / fp64: .to(int8) is a copy


def _parity_signs(rows: Tensor, cols: Tensor, dtype: torch.dtype) -> Tensor:
    """H[rows][:, cols] of Sylvester's matrix, (-1)^popcount(r & c)"""
    p = rows[:, None] & cols[None, :]
    for s in (8, 4, 2, 1):
        p = p ^ (p >> s)
    return (1 - 2 * (p & 1)).to(dtype)


def _core_factors(w: Tensor):
    """(s, C) as int8 when w = diag(s) . (C ⊗ H_{2^m})^T, the reference's random-hadamard matrix, with C of the order K its table
    gives for n = K * 2^m, else None.  The row signs and C are determined up to a sign per row block a; the rule fixed here takes
    s = w[:, 0] and C[c][a] = w[a 2^m][c 2^m] s[a 2^m] (so C[0][:] = 1).  The whole matrix is checked against them in row blocks."""
    n = w.size(0)
    k = table_core_order(n)
    m = n // k
    s = w[:, 0]
    if not bool(((s == 1) | (s == -1)).all()):
        return None
    core = (w[::m, ::m] * s[::m, None]).T.contiguous()
    if not bool(((core == 1) | (core == -1)).all()):
        return None
    log2_m = m.bit_length() - 1
    cols = torch.arange(n, device=w.device)
    block = max(1, (1 << 22) // n)
    for r0 in range(0, n, block):
        rows = torch.arange(r0, min(n, r0 + block), device=w.device)
        expected = (_parity_signs(rows & (m - 1), cols & (m - 1), w.dtype) * core[(cols >> log2_m)[None, :], (rows >> log2_m)[:, None]]
                    * s[r0:r0 + block, None])
        if not torch.equal(w[r0:r0 + block], expected):
            return None
    return s.to(torch.int8).contiguous(), core.to(torch.int8)


def _is_permutation(p: Tensor) -> bool:
    return p.dtype == torch.int64 and torch.equal(torch.sort(p).values, torch.arange(p.numel(), device=p.device))
