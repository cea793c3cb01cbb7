"""
Whole-model launches: every pack-quantized / naive-quantized module is compressed (or decompressed)
together with all other modules of the same (format, placement) group

  * tensors resident on one CUDA device  -> ONE multi-tensor kernel launch per kernel signature (ct_batched)
  * tensors resident in host memory      -> ONE pipelined H2D -> kernel -> D2H queue across all of them
                                            (ct_host_run_many); outputs land in host memory (pinned when
                                            the inputs are)

Results are bit-identical to the per-module plugin path (tests/test_gpu_compressors.py); modules that do
not qualify (other formats, activation ordering, N-D weights, meta tensors) take that path unchanged.

Modules offloaded to CPU or disk (offload/cache) are read where they are kept, without onloading: a CPUCache's pinned tensors
as they are, a DiskCache's files through `safe_open`.  They join the host-resident group, so a whole offloaded model is one
ct_host_run_many queue, and the results are written back through the module's cache as its new offloaded values (kept as they
are when pinned, new files for a DiskCache).  Offloaded modules that do not qualify take the per-module path, which onloads,
runs the kernels on the device and offloads the results.

What such a queue holds in host memory at once is bounded: a group with offloaded modules is cut into consecutive parts whose
outputs fit in `_host_budget()` (a quarter of the host memory available when the call starts), and each part is written back,
and its outputs released, before the next part is read.  A model under the budget is one queue.  Host queues run on the
modules' onload device.  Pinned outputs fall back to pageable memory when pinning fails.
"""
from __future__ import annotations

import logging
import os
from collections import defaultdict
from typing import Optional

import torch

from ... import _native as N
from ... import ops
from ...config import CompressionFormat
from ...offload.cache import CPUCache, DiskCache
from ...quantization import QuantizationScheme, QuantizationStatus
from ...utils.module import get_direct_state_dict, replace_direct_state_dict
from ..base import BaseCompressor, _resolve_format, compress_module, decompress_module

__all__ = ["compress_modules_batched", "decompress_modules_batched"]

_LOGGER = logging.getLogger(__name__)

_BATCHABLE = (CompressionFormat.pack_quantized, CompressionFormat.naive_quantized, CompressionFormat.int_quantized,
              CompressionFormat.float_quantized)
# fp4 nibble formats: one multi-tensor launch on CUDA placements, the cross-tensor host pipeline for host-resident modules
_FP4 = (CompressionFormat.nvfp4_pack_quantized, CompressionFormat.mxfp4_pack_quantized)


def _fp4_ok(sd, fmt, place, key: str) -> bool:
    if fmt not in _FP4 or place is None:
        return False
    if fmt == CompressionFormat.nvfp4_pack_quantized:
        gs = sd.get("weight_global_scale", None)
        t = sd.get(key)
        return gs is not None and gs.device == t.device and gs.dtype == torch.float32 and gs.numel() == 1 and gs.ndim >= 1
    return True


def _problem(c: "ops._Call", keep: list):
    """(desc, in, scale, zp, out) of one module's call, its output allocated where its input lives; `keep` holds the call (and the
    global scale its descriptor points at) until the launch"""
    out = _empty(c.out_shape, c.out_dtype, c.src)
    if c.p.gs is not None:
        c.desc.global_scale = c.p.gs.data_ptr()
    keep.append(c)
    return (c.desc, c.src.contiguous(), c.p.scale.contiguous(), c.p.zp.contiguous() if c.p.zp is not None else None, out)


def _compress_fp4_group(mods, fmt, place, force_format, host) -> None:
    comp = BaseCompressor.get_value_from_registry(fmt.value)
    probs, staged, keep = [], [], []
    for m in mods:
        scheme = m.quantization_scheme
        scheme.format = fmt
        sd = host.get(m) or get_direct_state_dict(m)
        gs = sd.get("weight_global_scale", None) if fmt == CompressionFormat.nvfp4_pack_quantized else None
        try:
            c = ops._quantize_pack_fp4_call(sd["weight"], sd["weight_scale"], sd.get("weight_zero_point", None), scheme.weights,
                                            global_scale=gs)
        except (ValueError, NotImplementedError):
            compress_module(m, force_format)
            continue
        probs.append(_problem(c, keep))
        staged.append((m, sd, probs[-1][4]))
    _run(N.OP_QUANTIZE_PACK_FP4, probs, place)
    for m, sd, out in staged:
        scheme = m.quantization_scheme
        new = sd.copy()
        new.pop("weight")
        new["weight_packed"] = out
        new["weight_scale"] = comp._compress_scale(sd["weight_scale"], scheme.weights)
        _write_back(m, comp._remove_symmetric_zp(new, scheme), host)
        m.quantization_status = QuantizationStatus.COMPRESSED


def _decompress_fp4_group(mods, fmt, place, force_format, host) -> None:
    comp = BaseCompressor.get_value_from_registry(fmt.value)
    dense = torch.bfloat16   # like the reference: unpack_fp4_from_uint8's default dtype (nvfp4/base.py:116)
    probs, staged, keep = [], [], []
    for m in mods:
        scheme = m.quantization_scheme
        scheme.format = fmt
        sd = host.get(m) or get_direct_state_dict(m)
        packed, sc = sd["weight_packed"], sd["weight_scale"]
        try:
            if sc.dtype not in (torch.float8_e4m3fn, torch.uint8):
                raise NotImplementedError   # only scales stored as the compressor writes them are batched
            c = ops._unpack_dequantize_fp4_call(packed, sc, sd.get("weight_global_scale", None), dense, comp._stored_scale)
        except (ValueError, NotImplementedError):
            decompress_module(m, force_format)
            continue
        probs.append(_problem(c, keep))
        new = sd.copy()
        new.pop("weight_packed")
        new["weight"] = probs[-1][4]
        new["weight_scale"] = comp._decompress_scale(sc, dense)
        staged.append((m, new))
    _run(N.OP_UNPACK_DEQUANTIZE_FP4, probs, place)
    for m, new in staged:
        _write_back(m, new, host)
        m.quantization_status = QuantizationStatus.DECOMPRESSED


def _host_state(module):
    """the direct tensors of a module offloaded to CPU or disk, read where they are kept (nothing is onloaded); None otherwise"""
    cache = module._parameters
    if not isinstance(cache, (CPUCache, DiskCache)) or not torch.cuda.is_available():
        return None
    out = {}
    for c in (cache, module._buffers):
        for name, t in c.offloaded_values.items():
            if isinstance(c, DiskCache):
                t = c.read(t, "cpu")
            out[name] = t.data if isinstance(t, (torch.nn.Parameter, torch.nn.Buffer)) else t
    return out


def _write_back(module, new: dict, host: dict) -> None:
    """replace the module's tensors; for an offloaded module, a tensor that went through unchanged keeps its offloaded value"""
    sd = host.get(module)
    if sd is not None:
        kept = {**module._buffers.offloaded_values, **module._parameters.offloaded_values}
        new = {k: (kept[k] if k in sd and v is sd[k] else v) for k, v in new.items()}
    replace_direct_state_dict(module, new)
    host.pop(module, None)   # the part is written back: its inputs are no longer needed


def _placement(sd, key: str):
    """('cuda', index) / ('cpu', None) when the module's streamed tensor and qparams share a placement, else None"""
    t, sc = sd.get(key, None), sd.get("weight_scale", None)
    if t is None or sc is None or t.ndim != 2 or t.device != sc.device or t.device.type not in ("cuda", "cpu"):
        return None
    zp = sd.get("weight_zero_point", None)
    if zp is not None and zp.device != t.device:
        return None
    g = sd.get("weight_g_idx", None)
    if g is not None and bool((g != -1).all()):
        return None  # activation ordering: per-module path
    if t.device.type == "cpu" and not torch.cuda.is_available():
        return None  # the per-module path raises the loud "no CUDA device" error
    return (t.device.type, t.device.index)


def _run(op: int, probs, place):
    if not probs:
        return
    if place[0] == "cuda":
        ops.batched(op, probs, place[1])
    else:
        ops.host_batched(op, probs, place[1])   # None: the current device


def _pinned_empty(shape, dtype) -> torch.Tensor:
    return torch.empty(shape, dtype=dtype, pin_memory=True)


_pin_failure_logged = False


def _empty(shape, dtype, like: torch.Tensor):
    global _pin_failure_logged
    if like.is_cuda:
        return torch.empty(shape, dtype=dtype, device=like.device)
    if like.is_pinned():
        try:
            return _pinned_empty(shape, dtype)
        except RuntimeError as e:
            if not _pin_failure_logged:
                _pin_failure_logged = True
                _LOGGER.warning("could not pin host memory for a compressor output (%s); using pageable memory", e)
    return torch.empty(shape, dtype=dtype)


def _host_budget() -> int:
    """bytes of outputs one host queue of offloaded modules may hold: a quarter of the host memory available now"""
    return os.sysconf("SC_AVPHYS_PAGES") * os.sysconf("SC_PAGE_SIZE") // 4


def _onload_index(module):
    """CUDA index of an offloaded module's onload device (None: the current device)"""
    device = torch.device(module._parameters.onload_device)
    return device.index if device.type == "cuda" else None


def _parts(groups, host, out_bytes):
    """the groups, with every host group that holds offloaded modules cut into consecutive parts whose outputs (estimated by
    `out_bytes(state)`) fit in the host budget; a module larger than the budget is a part of its own"""
    budget = None
    for key, mods in groups.items():
        if key[1][0] != "cpu" or not any(m in host for m in mods):
            yield key, mods
            continue
        if budget is None:
            budget = _host_budget()
        part, used = [], 0
        for m in mods:
            size = out_bytes(host.get(m) or m._parameters)
            if part and used + size > budget:
                yield key, part
                part, used = [], 0
            part.append(m)
            used += size
        if part:
            yield key, part


def _compressed_bytes(sd) -> int:
    return sd["weight"].nbytes   # every compressed form is at most as large as the dense weight


def _decompressed_bytes(sd) -> int:
    src = sd.get("weight_packed", None)
    if src is None:
        src = sd["weight"]
    per_byte = {torch.int32: 2, torch.uint8: 2}.get(src.dtype, 1) if "weight_packed" in sd else 1
    return src.nbytes * per_byte * max(2, sd["weight_scale"].element_size())


def _group(modules, force_format, key_of, fallback):
    """(format, placement) groups of the modules the batched path takes, and the host view of each offloaded one among them;
    every other module goes through `fallback` (the per-module path) right away"""
    groups, host = defaultdict(list), {}
    for m in modules:
        scheme = getattr(m, "quantization_scheme", None)
        if not isinstance(scheme, QuantizationScheme):
            continue
        fmt = _resolve_format(m, scheme, force_format)
        place, sd = None, None
        if fmt in _BATCHABLE + _FP4 and scheme.weights is not None:
            sd = _host_state(m)
            view, key = (sd if sd is not None else m._parameters), key_of(fmt)
            place = _placement(view, key)
            if place is not None and not (fmt in _BATCHABLE or _fp4_ok(view, fmt, place, key)):
                place = None
            if place is not None and sd is not None:
                place = ("cpu", _onload_index(m))
        if place is None:
            fallback(m, force_format)
            continue
        groups[(fmt, place)].append(m)
        if sd is not None:
            host[m] = sd
    return groups, host


def compress_modules_batched(modules, force_format: Optional[CompressionFormat] = None) -> None:
    groups, host = _group(modules, force_format, lambda fmt: "weight", compress_module)
    for (fmt, place), mods in _parts(groups, host, _compressed_bytes):
        if fmt in _FP4:
            _compress_fp4_group(mods, fmt, place, force_format, host)
            continue
        comp = BaseCompressor.get_value_from_registry(fmt.value)
        pack = fmt == CompressionFormat.pack_quantized
        probs, staged, keep = [], [], []
        for m in mods:
            scheme = m.quantization_scheme
            scheme.format = fmt
            args = scheme.weights
            sd = host.get(m) or get_direct_state_dict(m)
            w, sc = sd["weight"], sd["weight_scale"]
            # the zero point goes through like in the per-module plugin path (ops.quantize): for integer codes a symmetric
            # scheme's all-zero zero point cannot change a code (x/s + 0 only turns -0.0 into +0.0, which rounds to the same
            # integer), so it is skipped; for fp8 codes -0.0 and +0.0 are different bytes (0x80 / 0x00), so it is added
            zp = sd.get("weight_zero_point", None) if (not args.symmetric or args.type == "float") else None
            try:
                c = ops._quantize_pack_call(w, sc, zp, args) if pack else ops._quantize_call(w, sc, zp, args, dtype=args.pytorch_dtype())
            except (ValueError, NotImplementedError):
                compress_module(m, force_format)
                continue
            probs.append(_problem(c, keep))
            staged.append((m, sd, probs[-1][4]))
        _run(N.OP_QUANTIZE_PACK if pack else N.OP_QUANTIZE, probs, place)
        for m, sd, out in staged:
            scheme = m.quantization_scheme
            args = scheme.weights
            new = sd.copy()
            w = new.pop("weight")
            if pack:
                new["weight_packed"] = out
                new["weight_shape"] = torch.tensor(w.shape)
                if not args.symmetric and args.strategy in ("group", "channel"):
                    new["weight_zero_point"] = ops.pack_to_int32(sd["weight_zero_point"], args.num_bits, packed_dim=0).contiguous()
            else:
                new["weight"] = out
            new = comp._remove_symmetric_zp(new, scheme)
            _write_back(m, new, host)
            m.quantization_status = QuantizationStatus.COMPRESSED


def decompress_modules_batched(modules, force_format: Optional[CompressionFormat] = None) -> None:
    packed = (CompressionFormat.pack_quantized,) + _FP4
    groups, host = _group(modules, force_format, lambda fmt: "weight_packed" if fmt in packed else "weight", decompress_module)
    for (fmt, place), mods in _parts(groups, host, _decompressed_bytes):
        if fmt in _FP4:
            _decompress_fp4_group(mods, fmt, place, force_format, host)
            continue
        pack = fmt == CompressionFormat.pack_quantized
        probs, staged, keep = [], [], []
        for m in mods:
            scheme = m.quantization_scheme
            scheme.format = fmt
            args = scheme.weights
            sd = host.get(m) or get_direct_state_dict(m)
            sc = sd["weight_scale"]
            zp = sd.get("weight_zero_point", None)
            new = sd.copy()
            try:
                if pack:
                    shape = tuple(int(v) for v in sd["weight_shape"].tolist())
                    if zp is not None and not args.symmetric and args.strategy in ("group", "channel"):
                        zp = ops.unpack_from_int32(zp, args.num_bits, (*shape[:-1], sc.shape[-1]), packed_dim=0)
                        new["weight_zero_point"] = zp
                    c = ops._unpack_dequantize_call(sd["weight_packed"], sc, zp, args.num_bits, shape)
                    new.pop("weight_packed")
                else:
                    c = ops._dequantize_call(sd["weight"], sc, zp)
            except (ValueError, NotImplementedError):
                decompress_module(m, force_format)
                continue
            probs.append(_problem(c, keep))
            new["weight"] = probs[-1][4]
            staged.append((m, new))
        _run(N.OP_UNPACK_DEQUANTIZE if pack else N.OP_DEQUANTIZE, probs, place)
        for m, new in staged:
            _write_back(m, new, host)
            m.quantization_status = QuantizationStatus.DECOMPRESSED
