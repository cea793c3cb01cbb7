"""
Write fences around every device entry point of include/ct_b200.h: each output lies between 64 KiB guards of poison inside a larger
buffer, each input between guards of NaN / the largest finite value (0x77 for integer data), and each case runs twice with two poisons
(helpers and rationale: tests/test_write_fences_host.py).  A store past the end of an output, an output element that is never written
and a write into an input all fail with the entry point, the case and the byte offset.  Over-reads that neither fault nor change a result
(a vector load past the end whose extra lanes are discarded) cannot be seen this way and are not looked for.

Case ids name the dispatch path each shape takes (`fast`, `generic`, `lookback`, `twophase`, ...) and the predicate boundary it sits on.
Outputs are compared with the oracle where it restates the op (pack / unpack, the quantize family, bitmasks, 2:4, semi-structured, FP4
and MX pieces, AutoAWQ); the fused observers, FP4 compressors, dynamic activations, strided K / V and the device Walsh-Hadamard are
compared with the same entry point run on plain tensors through the public op, which the rest of the suite ties to the oracle.

ENTRY_TESTS maps every `ct_*` function with a non-const pointer parameter to the tests that fence it;
test_every_writing_entry_point_is_fenced parses the header and fails on any function that is neither there nor in EXEMPT.
"""
from __future__ import annotations

import ctypes
import math
import re
from pathlib import Path

import pytest
import torch

import oracle
from compressed_tensors_b200 import _native as N
from compressed_tensors_b200 import ops
from tests.test_write_fences_host import (G, POISONS, Fence, FencedInput, fenced, in_guard, qproblem, quant_call, quant_desc, quant_io,
                                          QUANT_FNS, run_fenced)

DEV = "cuda:0"
HEADER = Path(__file__).resolve().parent.parent / "include" / "ct_b200.h"

# functions with a non-const pointer parameter that write no tensor
EXEMPT = {
    "ct_selftest_division": "writes one host mismatch counter; an exhaustive device self-test, not a tensor op",
    "ct_selftest_fp4_division": "writes one host mismatch counter; an exhaustive device self-test, not a tensor op",
}

ENTRY_TESTS = {
    "ct_pack_int32": ["test_pack_unpack_int32"],
    "ct_unpack_int32": ["test_pack_unpack_int32"],
    "ct_quantize": ["test_quantize_family"],
    "ct_dequantize": ["test_quantize_family"],
    "ct_fake_quantize": ["test_quantize_family"],
    "ct_quantize_pack_int32": ["test_quantize_family"],
    "ct_unpack_dequantize_int32": ["test_quantize_family"],
    "ct_fake_quantize_heads": ["test_strided_kv_views"],
    "ct_hadamard_transform": ["test_hadamard_transform", "test_strided_kv_views"],
    "ct_observe_quantize_pack_int32": ["test_observers"],
    "ct_observe_quantize_channel": ["test_channel_observer_cluster_shapes"],
    "ct_observe_tensor": ["test_observers"],
    "ct_observe_quantize_tensor": ["test_observers"],
    "ct_observe_quantize_block": ["test_observers"],
    "ct_observe_quantize_mx": ["test_observers"],
    "ct_observe_quantize_pack_nvfp4": ["test_observers"],
    "ct_dynamic_fake_quantize": ["test_dynamic_fake_quantize"],
    "ct_cast_to_fp4": ["test_fp4_pieces"],
    "ct_pack_fp4": ["test_fp4_pieces"],
    "ct_unpack_fp4": ["test_fp4_pieces"],
    "ct_mx_scale_compress": ["test_fp4_pieces"],
    "ct_mx_scale_decompress": ["test_fp4_pieces"],
    "ct_quantize_pack_fp4": ["test_fp4_compressors"],
    "ct_unpack_dequantize_fp4": ["test_fp4_compressors"],
    "ct_awq_repack_int4": ["test_awq_repack"],
    "ct_awq_repack_zeros_int4": ["test_awq_repack"],
    "ct_pack_bitmasks": ["test_bitmasks_and_24"],
    "ct_unpack_bitmasks": ["test_bitmasks_and_24"],
    "ct_sparse24_compress": ["test_bitmasks_and_24"],
    "ct_sparse24_decompress": ["test_bitmasks_and_24"],
    "ct_bitmask_count": ["test_bitmask_unstructured"],
    "ct_bitmask_compress": ["test_bitmask_unstructured"],
    "ct_bitmask_decompress": ["test_bitmask_unstructured"],
    "ct_bitmask_compress_onepass": ["test_bitmask_unstructured"],
    "ct_sparse24_quantize_pack_int4": ["test_sparse24_int4"],
    "ct_sparse24_unpack_dequantize_int4": ["test_sparse24_int4"],
    "ct_semi_structured_from_dense": ["test_semi_structured"],
    "ct_semi_structured_to_dense": ["test_semi_structured"],
    "ct_batched": ["test_batched_arena", "test_batched_arena_dynamic_and_graph"],
    "ct_host_run_many": ["test_host_run_many"],
}


def _header_functions():
    """{name: [parameter declarations]} of every function declared in the header"""
    text = re.sub(r"/\*.*?\*/", "", HEADER.read_text(), flags=re.S)
    out = {}
    for m in re.finditer(r"^\s*(?:const\s+)?[\w]+\s*\*?\s*(ct_\w+)\s*\(([^)]*)\)\s*;", text, flags=re.M):
        out[m.group(1)] = [p.strip() for p in m.group(2).split(",") if p.strip() and p.strip() != "void"]
    return out


def test_every_writing_entry_point_is_fenced():
    funcs = _header_functions()
    assert "ct_batched" in funcs and "ct_version" in funcs, "the header parser found no declarations"
    writing = {f for f, params in funcs.items() if any("*" in p and not p.startswith("const ") for p in params)}
    missing = sorted(writing - set(ENTRY_TESTS) - set(EXEMPT))
    assert not missing, f"entry points with a non-const pointer parameter and no write fence: {missing}"
    stale = sorted((set(ENTRY_TESTS) | set(EXEMPT)) - set(funcs))
    assert not stale, f"table rows for functions the header does not declare: {stale}"
    assert all(EXEMPT.values())
    names = set(globals())
    for f, tests in ENTRY_TESTS.items():
        assert tests and all(t in names for t in tests), f"{f}: {tests}"
    ops_in_header = re.search(r"typedef enum ct_batch_op_t \{(.*?)\}", HEADER.read_text(), flags=re.S).group(1)
    header_ops = set(re.findall(r"(CT_OP_\w+)\s*=", ops_in_header))
    assert header_ops == {f"CT_OP_{k}" for k in BATCH_OPS}, "every ct_batch_op_t runs in the batched arena"


def _st():
    return N.stream_ptr(0)


def _launches(fn):
    before = N.launch_count()
    fn()
    return N.launch_count() - before


# ------------------------------------------------------------------------------------------------------------------------------
# pack / unpack: plan_bits (4 / 8 bits, (cols*bits) % 32 == 0, n % unit == 0, 16-byte aligned) or the generic kernels
# ------------------------------------------------------------------------------------------------------------------------------
def _pack_shapes(bits):
    shapes = [(1, 37, "generic-ragged"), (3, 100, "generic-cols%8"), (1, 1, "generic-one")]
    if bits in (4, 8):
        unit = 16
        shapes += [(1, unit * 2, "fast-one-chunk"), (1, unit * 1023, "fast-tile-1"), (1, unit * 1024, "fast-tile"),
                   (2, unit * 1025 // 2 * 2 // 2, "fast-tile+1"), (1, unit * 2049, "fast-2tile+1")]
    return shapes


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [256, 16, 4])
@pytest.mark.parametrize("bits", range(1, 9))
def test_pack_unpack_int32(bits, offset):
    lib = N.lib()
    for rows, cols, path in _pack_shapes(bits):
        g = torch.Generator().manual_seed(bits * 1000 + cols)
        codes = torch.randint(-(1 << (bits - 1)), 1 << (bits - 1), (rows, cols), generator=g, dtype=torch.int8)
        packed = oracle.pack_to_int32(codes, bits)
        if offset == 4:
            path = "generic-misaligned"
        case = f"{path}-bits{bits}-{rows}x{cols}-off{offset}"
        run_fenced("ct_pack_int32", case, {"x": codes}, {"out": (tuple(packed.shape), torch.int32)},
                   lambda i, o: lib.ct_pack_int32(N.ptr(i["x"]), N.ptr(o["out"]), rows, cols, bits, 1, 0, _st()),
                   {"out": packed}, offset=offset, device=DEV)
        run_fenced("ct_unpack_int32", case, {"x": packed}, {"out": ((rows, cols), torch.int8)},
                   lambda i, o: lib.ct_unpack_int32(N.ptr(i["x"]), N.ptr(o["out"]), rows, cols, bits, 1, 0, _st()),
                   {"out": codes}, offset=offset, device=DEV)
        p0 = oracle.pack_to_int32(codes, bits, 0)
        run_fenced("ct_pack_int32", case + "-dim0", {"x": codes}, {"out": (tuple(p0.shape), torch.int32)},
                   lambda i, o: lib.ct_pack_int32(N.ptr(i["x"]), N.ptr(o["out"]), rows, cols, bits, 0, 0, _st()),
                   {"out": p0}, offset=offset, device=DEV)


# ------------------------------------------------------------------------------------------------------------------------------
# the quantize family: plan_one.  bf16 quantize / dequantize / quantize+pack / unpack+dequantize run on 2048-chunk tiles, fake_quantize
# and fp32 on 1024-chunk tiles; a chunk is 8 elements.  cols % 8 != 0 and misaligned pointers take the generic kernels.
# ------------------------------------------------------------------------------------------------------------------------------
QFAMILY = [
    # (strategy, rows, cols, group, block, dtype, bits, path)
    ("tensor", 1, 8, None, None, torch.bfloat16, 8, "fast-one-chunk"),
    ("tensor", 1, 8 * 2047, None, None, torch.bfloat16, 8, "fast-2048tile-1"),
    ("tensor", 1, 8 * 2048, None, None, torch.bfloat16, 8, "fast-2048tile"),
    ("tensor", 1, 8 * 2049, None, None, torch.bfloat16, 8, "fast-2048tile+1-last16B"),
    ("channel", 1, 8 * 1023, None, None, torch.float32, 8, "fast-1024tile-1"),
    ("channel", 2, 8 * 512, None, None, torch.float32, 8, "fast-1024tile"),
    ("channel", 1, 8 * 1025, None, None, torch.float32, 8, "fast-1024tile+1"),
    ("group", 3, 8 * 33 * 4, 32 * 33 // 33, None, torch.bfloat16, 4, "fast-group-units%G"),
    ("group", 5, 8 * 128 + 128, 128, None, torch.float16, 4, "fast-group"),
    ("channel", 7, 37, None, None, torch.bfloat16, 8, "generic-cols%8"),
    ("channel", 3, 8 * 13 + 4, None, None, torch.bfloat16, 8, "generic-cols%32"),
    ("group", 2, 8 * 16 + 64, 64, None, torch.bfloat16, 4, "fast-cols%128"),
    ("block", 37, 70, None, (16, 32), torch.bfloat16, 8, "generic-block-ragged"),
    ("block", 130, 264, None, (128, 128), torch.bfloat16, 8, "fast2d-block-ragged"),
]


def _fid(c):
    return f"{c[7]}-{c[0]}-{c[1]}x{c[2]}-{str(c[5])[6:]}"


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [256, 16, 2])
@pytest.mark.parametrize("op", list(QUANT_FNS))
@pytest.mark.parametrize("c", QFAMILY, ids=_fid)
def test_quantize_family(c, op, offset):
    strategy, rows, cols, gs, blk, dt, bits, path = c
    if op in ("quantize_pack", "unpack_dequantize"):
        bits = 4
    if offset == 2 and op in ("quantize_pack", "unpack_dequantize"):
        offset = 4          # int32 words: 4-byte aligned at least; plan_one sends anything not 16-byte aligned to the generic kernel
    if offset % torch.empty((), dtype=dt).element_size():
        pytest.skip("an fp32 tensor is 4-byte aligned at least")
    x, scale, zp, args = qproblem(strategy, rows, cols, dt, bits, "int", asym=True, group_size=gs, block=blk, seed=len(path))
    d, want = quant_desc(op, x, scale, zp, args)
    ins, outs = quant_io(op, x, scale, zp, args, want)
    run_fenced(QUANT_FNS[op], f"{path if offset >= 16 else 'generic-misaligned'}-{_fid(c)}-off{offset}", ins, outs,
               quant_call(op, d, 0, _st()), {"out": want}, offset=offset, device=DEV)


# ------------------------------------------------------------------------------------------------------------------------------
# observers: outputs compared with the public op on plain tensors
# ------------------------------------------------------------------------------------------------------------------------------
def _x(rows, cols, dtype=torch.bfloat16, seed=0):
    g = torch.Generator().manual_seed(seed + rows * 131 + cols)
    return (torch.randn(rows, cols, generator=g) * 3).to(dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [256, 16])
def test_observers(offset):
    from types import SimpleNamespace as NS

    lib = N.lib()
    # fused group observer + pack: rows * cols % 32 == 0, groups of 32 * {1, 2, 4, 8}
    for rows, cols, group, bits in ((1, 32, 32, 4), (3, 96, 32, 8), (5, 8 * 2049 // 32 * 32, 256, 4), (2, 128 * 3, 128, 4)):
        x = _x(rows, cols)
        args = NS(strategy="group", group_size=group, num_bits=bits, type="int", symmetric=False)
        want_p, want_s, want_z = ops.observe_quantize_pack(x.to(DEV), args)
        d = N.QuantDesc()
        d.rows, d.cols, d.rdiv, d.cdiv, d.s_row_stride = rows, cols, 1, group, cols // group
        d.x_dtype = d.scale_dtype = d.compute_dtype = N.DT[x.dtype]
        d.zp_dtype, d.q_dtype, d.out_dtype, d.qtype, d.num_bits = N.DT[torch.int8], N.DT[torch.int8], N.DT_NONE, N.Q_INT, bits
        run_fenced("ct_observe_quantize_pack_int32", f"fast-g{group}-{rows}x{cols}-off{offset}", {"x": x},
                   {"s": (tuple(want_s.shape), x.dtype), "z": (tuple(want_z.shape), torch.int8), "p": (tuple(want_p.shape), torch.int32)},
                   lambda i, o: lib.ct_observe_quantize_pack_int32(ctypes.byref(d), N.ptr(i["x"]), N.ptr(o["s"]), N.ptr(o["z"]), N.ptr(o["p"]), 0, _st()),
                   {"s": want_s, "z": want_z, "p": want_p}, offset=offset, device=DEV)
    # per-tensor observer, alone and fused with quantize
    for rows, cols in ((1, 8), (3, 8 * 2049), (64, 8 * 4096 + 8)):
        x = _x(rows, cols, seed=1)
        xd = x.to(DEV)
        args = NS(strategy="tensor", num_bits=8, type="int", symmetric=False, group_size=None)
        want_s, want_z = ops.observe_tensor_qparams(xd, args)
        d = ops._tensor_desc(xd, N.Q_INT, 8, asym=True)
        run_fenced("ct_observe_tensor", f"{rows}x{cols}-off{offset}", {"x": x}, {"s": ((1,), x.dtype), "z": ((1,), torch.int8)},
                   lambda i, o: lib.ct_observe_tensor(ctypes.byref(d), N.ptr(i["x"]), 0, N.ptr(o["s"]), N.ptr(o["z"]), 0, _st()),
                   {"s": want_s, "z": want_z}, offset=offset, device=DEV)
        want_q, want_s, want_z = ops.observe_quantize(xd, args)
        d = ops._tensor_desc(xd, N.Q_INT, 8, q_dt=torch.int8, asym=True)
        run_fenced("ct_observe_quantize_tensor", f"{rows}x{cols}-off{offset}", {"x": x},
                   {"s": ((1,), x.dtype), "z": ((1,), torch.int8), "q": ((rows, cols), torch.int8)},
                   lambda i, o: lib.ct_observe_quantize_tensor(ctypes.byref(d), N.ptr(i["x"]), N.ptr(o["s"]), N.ptr(o["z"]), N.ptr(o["q"]), 0, _st()),
                   {"s": want_s, "z": want_z, "q": want_q}, offset=offset, device=DEV)
    # FP8_BLOCK with ragged edge blocks, MXFP4 / MXFP8
    for rows, cols, bh, bw in ((1, 8, 128, 128), (130, 264, 128, 128), (37, 72, 16, 32), (3, 8 * 129, 1, 64)):
        x = _x(rows, cols, seed=2)
        want_q, want_s = ops.observe_quantize(x.to(DEV), NS(strategy="block", block_structure=[bh, bw], num_bits=8, type="float",
                                                            symmetric=True, group_size=None))[:2]
        d = ops._block_desc(rows, cols, bh, bw, x.dtype)
        run_fenced("ct_observe_quantize_block", f"block{bh}x{bw}-{rows}x{cols}-off{offset}", {"x": x},
                   {"s": (tuple(want_s.shape), x.dtype), "q": ((rows, cols), torch.float8_e4m3fn)},
                   lambda i, o: lib.ct_observe_quantize_block(ctypes.byref(d), N.ptr(i["x"]), N.ptr(o["s"]), N.ptr(o["q"]), 0, _st()),
                   {"s": want_s.reshape(-1), "q": want_q}, offset=offset, device=DEV)
    for rows, cols, bits in ((1, 32, 4), (3, 96, 8), (33, 32 * 65, 4)):
        x = _x(rows, cols, seed=3)
        want_q, want_s = ops.observe_quantize_mx(x.to(DEV), NS(strategy="group", group_size=32, num_bits=bits, type="float",
                                                                 symmetric=True, scale_dtype=torch.uint8, block_structure=None))
        d = ops._mx_desc(rows, cols, bits, x.dtype)
        run_fenced("ct_observe_quantize_mx", f"mx{bits}-{rows}x{cols}-off{offset}", {"x": x},
                   {"s": (tuple(want_s.shape), want_s.dtype), "q": (tuple(want_q.shape), want_q.dtype)},
                   lambda i, o: lib.ct_observe_quantize_mx(ctypes.byref(d), N.ptr(i["x"]), N.ptr(o["s"]), N.ptr(o["q"]), 0, _st()),
                   {"s": want_s, "q": want_q}, offset=offset, device=DEV)
    # NVFP4 observer + pack, given the global scale
    for rows, cols in ((1, 32), (5, 32 * 129)):
        x = _x(rows, cols, seed=4)
        args = NS(strategy="tensor_group", group_size=16, num_bits=4, type="float", symmetric=True)
        gsc = torch.tensor([448 * 6 / float(x.float().abs().max())], dtype=torch.float32)
        want_p, want_s, _ = ops.observe_quantize_pack_nvfp4(x.to(DEV), args, gsc.to(DEV))

        def call(i, o, rows=rows, cols=cols, x=x):
            d = N.QuantDesc()
            d.rows, d.cols, d.rdiv, d.cdiv, d.s_row_stride = rows, cols, 1, 16, cols // 16
            d.x_dtype, d.scale_dtype, d.compute_dtype = N.DT[x.dtype], N.DT[torch.float8_e4m3fn], N.DT[torch.float32]
            d.zp_dtype, d.q_dtype, d.out_dtype, d.qtype, d.num_bits = N.DT_NONE, N.DT[x.dtype], N.DT_NONE, N.Q_FP4, 4
            d.global_scale, d.seff_dtype = i["gs"].data_ptr(), N.DT[torch.float32]
            return lib.ct_observe_quantize_pack_nvfp4(ctypes.byref(d), N.ptr(i["x"]), N.ptr(o["s"]), N.ptr(o["p"]), 0, _st())

        run_fenced("ct_observe_quantize_pack_nvfp4", f"fast-{rows}x{cols}-off{offset}", {"x": x, "gs": gsc},
                   {"s": (tuple(want_s.shape), want_s.dtype), "p": (tuple(want_p.shape), torch.uint8)}, call,
                   {"s": want_s, "p": want_p}, offset=offset, device=DEV)


# the cluster-wide channel observer: a row of `units` 16-byte units is split over the ranks of a cluster (chan_cluster_shape), the last
# slice short; rows fewer than the resident clusters and many more
CHANNEL_COLS = [8, 8 * 1023, 16384] + [16384 * k + 8 for k in range(1, 8)] + [8 * 16384]


@pytest.mark.gpu
@pytest.mark.parametrize("cols", CHANNEL_COLS)
def test_channel_observer_cluster_shapes(cols):
    from types import SimpleNamespace as NS

    lib = N.lib()
    for rows, pack in ((3, False), (300 if cols <= 16384 else 40, True)):
        x = _x(rows, cols, seed=5)
        bits = 4 if pack else 8
        args = NS(strategy="channel", num_bits=bits, type="int", symmetric=False, group_size=None)
        want_q, want_s, want_z = ops.observe_quantize(x.to(DEV), args, pack=pack)
        qdt = torch.int32 if pack else torch.int8
        d = N.QuantDesc()
        d.rows, d.cols, d.rdiv, d.cdiv, d.s_row_stride = rows, cols, 1, N.INF, 1
        d.x_dtype = d.scale_dtype = d.compute_dtype = N.DT[x.dtype]
        d.zp_dtype, d.q_dtype, d.out_dtype, d.qtype, d.num_bits = N.DT[torch.int8], N.DT[qdt], N.DT_NONE, N.Q_INT, bits
        outs = {"s": ((rows, 1), x.dtype), "z": ((rows, 1), torch.int8), "q": (tuple(want_q.shape), qdt)}
        case = f"{'pack4' if pack else 'int8'}-{rows}x{cols}"

        def call(i, o):
            rc = lib.ct_observe_quantize_channel(ctypes.byref(d), N.ptr(i["x"]), N.ptr(o["s"]), N.ptr(o["z"]), N.ptr(o["q"]), 0, _st())
            if rc == N.CT_E_UNSUPPORTED:       # a row wider than one cluster holds: declined, nothing written
                o["q"].copy_(want_q); o["s"].copy_(want_s); o["z"].copy_(want_z)
                return N.CT_OK
            return rc

        run_fenced("ct_observe_quantize_channel", case, {"x": x}, outs, call, {"s": want_s, "z": want_z, "q": want_q}, device=DEV)


# ------------------------------------------------------------------------------------------------------------------------------
# dynamic activations: TOKEN / GROUP / TENSOR with int, fp8 and MX scales
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("offset", [256, 16])
def test_dynamic_fake_quantize(offset):
    from types import SimpleNamespace as NS

    lib = N.lib()
    cases = [
        ("token", None, 8, "int", False, None, torch.int8, (1, 8)),
        ("token", None, 8, "int", False, None, torch.int8, (37, 8 * 129)),
        ("token", None, 8, "float", True, None, torch.float8_e4m3fn, (5, 8 * 4097)),
        ("group", 16, 4, "int", False, None, torch.int8, (3, 16 * 7)),
        ("group", 128, 8, "int", True, None, torch.int8, (9, 128 * 33)),
        ("group", 32, 4, "float", True, torch.uint8, torch.uint8, (7, 32 * 5)),
        ("tensor", None, 8, "int", False, None, torch.int8, (3, 8 * 2049)),
    ]
    for strategy, group, bits, qt, sym, sdt, zdt, (rows, cols) in cases:
        x = _x(rows, cols, seed=6)
        args = NS(strategy=strategy, group_size=group, num_bits=bits, type=qt, symmetric=sym, scale_dtype=sdt, zp_dtype=zdt,
                  block_structure=None)
        got = ops.dynamic_fake_quantize(x.to(DEV), args)
        assert got is not None, (strategy, group, bits, qt)
        want_o, want_s, want_z = got
        r, c, rdiv, cdiv, srs, sshape = ops._dynamic_layout(x, args)
        qtype, nb = ops._qparams(args)
        d = N.QuantDesc()
        d.rows, d.cols, d.rdiv, d.cdiv, d.s_row_stride = r, c, rdiv, cdiv, srs
        d.x_dtype = d.out_dtype = N.DT[x.dtype]
        d.scale_dtype, d.zp_dtype, d.compute_dtype, d.seff_dtype = N.DT[x.dtype], N.DT[zdt], N.DT[x.dtype], N.DT[x.dtype]
        d.q_dtype, d.qtype, d.num_bits = N.DT_NONE, qtype, nb
        sarg = ops._SCALE_ROUNDING[sdt]
        run_fenced("ct_dynamic_fake_quantize", f"{strategy}{group or ''}-{qt}{bits}-{rows}x{cols}-off{offset}", {"x": x},
                   {"o": ((rows, cols), x.dtype), "s": (tuple(want_s.shape), x.dtype), "z": (tuple(want_z.shape), zdt)},
                   lambda i, o: lib.ct_dynamic_fake_quantize(ctypes.byref(d), int(not sym), sarg, N.ptr(i["x"]), N.ptr(o["o"]),
                                                              N.ptr(o["s"]), N.ptr(o["z"]), 0, _st()),
                   {"o": want_o, "s": want_s, "z": want_z}, offset=offset, device=DEV)


# ------------------------------------------------------------------------------------------------------------------------------
# FP4 / MX pieces (oracle) and compressors (public op)
# ------------------------------------------------------------------------------------------------------------------------------
def _fp4_values(rows, cols, dtype, seed=0):
    g = torch.Generator().manual_seed(seed + cols)
    grid = torch.tensor([0, .5, 1, 1.5, 2, 3, 4, 6, -0., -.5, -1, -1.5, -2, -3, -4, -6])
    return grid[torch.randint(0, 16, (rows, cols), generator=g)].to(dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [256, 16, 2])
def test_fp4_pieces(offset):
    lib = N.lib()
    for rows, cols in ((1, 2), (3, 34), (1, 8 * 2049), (7, 16 * 33)):
        x = (torch.randn(rows, cols, generator=torch.Generator().manual_seed(cols)) * 3).bfloat16()
        n = rows * cols
        run_fenced("ct_cast_to_fp4", f"{rows}x{cols}-off{offset}", {"x": x}, {"o": ((rows, cols), x.dtype)},
                   lambda i, o: lib.ct_cast_to_fp4(N.ptr(i["x"]), N.DT[x.dtype], N.ptr(o["o"]), n, 0, _st()),
                   {"o": oracle.cast_to_fp4(x)}, offset=offset, device=DEV)
        v = _fp4_values(rows, cols, torch.bfloat16)
        packed = oracle.pack_fp4_to_uint8(v)
        run_fenced("ct_pack_fp4", f"{rows}x{cols}-off{offset}", {"x": v}, {"o": (tuple(packed.shape), torch.uint8)},
                   lambda i, o: lib.ct_pack_fp4(N.ptr(i["x"]), N.DT[v.dtype], N.ptr(o["o"]), rows, cols, 0, _st()),
                   {"o": packed}, offset=offset, device=DEV)
        run_fenced("ct_unpack_fp4", f"{rows}x{cols}-off{offset}", {"x": packed}, {"o": ((rows, cols), torch.bfloat16)},
                   lambda i, o: lib.ct_unpack_fp4(N.ptr(i["x"]), N.ptr(o["o"]), N.DT[torch.bfloat16], rows, cols, 0, _st()),
                   {"o": oracle.unpack_fp4_from_uint8(packed, rows, cols, torch.bfloat16)}, offset=offset, device=DEV)
        s = torch.rand(rows, cols, generator=torch.Generator().manual_seed(n)).bfloat16() * 2 ** 10 + 2 ** -10
        e = oracle.compress_mx_scale(s)
        run_fenced("ct_mx_scale_compress", f"{rows}x{cols}-off{offset}", {"x": s}, {"o": ((rows, cols), torch.uint8)},
                   lambda i, o: lib.ct_mx_scale_compress(N.ptr(i["x"]), N.DT[s.dtype], N.ptr(o["o"]), n, 0, _st()),
                   {"o": e}, offset=offset, device=DEV)
        run_fenced("ct_mx_scale_decompress", f"{rows}x{cols}-off{offset}", {"x": e}, {"o": ((rows, cols), torch.bfloat16)},
                   lambda i, o: lib.ct_mx_scale_decompress(N.ptr(i["x"]), N.ptr(o["o"]), n, 0, _st()),
                   {"o": oracle.decompress_mx_scale(e)}, offset=offset, device=DEV)


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [256, 16, 2])
def test_fp4_compressors(offset):
    from types import SimpleNamespace as NS

    lib = N.lib()
    for rows, cols, group in ((1, 32, 32), (3, 32 * 65, 32), (5, 16 * 3, 16), (2, 32 * 2049, 16)):
        x = _x(rows, cols, seed=7)
        args = NS(strategy="group", group_size=group, num_bits=4, type="float")
        amax = x.float().unflatten(-1, (-1, group)).abs().amax(-1)
        scale = (amax / 6 + 2 ** -8).to(x.dtype)
        want = ops.quantize_pack_fp4(x.to(DEV), scale.to(DEV), None, args)
        p = ops._resolve(x, scale, None, args, None)
        d = ops._desc(p, x.dtype, scale.dtype, None, x.dtype, x.dtype, None, N.Q_FP4, 4, scale.dtype)
        path = ("fast" if cols % 32 == 0 and group % 32 == 0 else "generic") if offset >= 16 else "generic-misaligned"
        run_fenced("ct_quantize_pack_fp4", f"{path}-g{group}-{rows}x{cols}-off{offset}", {"x": x, "s": scale},
                   {"o": (tuple(want.shape), torch.uint8)},
                   lambda i, o: lib.ct_quantize_pack_fp4(ctypes.byref(d), N.ptr(i["x"]), N.ptr(i["s"]), None, None, N.ptr(o["o"]), 0, _st()),
                   {"o": want}, offset=offset, device=DEV)
        want_d = ops.unpack_dequantize_fp4(want, scale.to(DEV), dtype=x.dtype)
        d2 = ops._desc(p, None, scale.dtype, None, None, None, x.dtype, N.Q_FP4, 4, scale.dtype)
        run_fenced("ct_unpack_dequantize_fp4", f"{path}-g{group}-{rows}x{cols}-off{offset}", {"p": want.cpu(), "s": scale},
                   {"o": ((rows, cols), x.dtype)},
                   lambda i, o: lib.ct_unpack_dequantize_fp4(ctypes.byref(d2), N.ptr(i["p"]), N.ptr(i["s"]), None, None, N.ptr(o["o"]), 0, _st()),
                   {"o": want_d}, offset=offset, device=DEV)


# ------------------------------------------------------------------------------------------------------------------------------
# AutoAWQ repack: 32-byte row stores need KW % 4 == 0 AND a 16-byte aligned output; a 4-byte aligned one takes the scalar stores
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("offset", [256, 16, 4])
def test_awq_repack(offset):
    lib = N.lib()
    for k, n in ((1, 8), (64, 256), (96, 264), (130, 512), (7, 8 * 33)):
        g = torch.Generator().manual_seed(k * n)
        qw = torch.randint(-2 ** 31, 2 ** 31 - 1, (k, n // 8), generator=g, dtype=torch.int32)
        want = oracle.awq_repack(qw)
        kw = (k + 7) // 8
        path = ("vec32B" if kw % 4 == 0 else "scalar") if offset >= 16 else "scalar-misaligned"
        run_fenced("ct_awq_repack_int4", f"{path}-K{k}-N{n}-off{offset}", {"x": qw}, {"o": (tuple(want.shape), torch.int32)},
                   lambda i, o: lib.ct_awq_repack_int4(N.ptr(i["x"]), N.ptr(o["o"]), k, n, 0, _st()), {"o": want},
                   offset=offset, device=DEV)
        wz = oracle.awq_repack_zeros(qw)
        run_fenced("ct_awq_repack_zeros_int4", f"G{k}-N{n}-off{offset}", {"x": qw}, {"o": (tuple(wz.shape), torch.int32)},
                   lambda i, o: lib.ct_awq_repack_zeros_int4(N.ptr(i["x"]), N.ptr(o["o"]), k, n, 0, _st()), {"o": wz},
                   offset=offset, device=DEV)


# ------------------------------------------------------------------------------------------------------------------------------
# bitmasks, 2:4, unstructured (vec16_ok, bitmask_lookback_ok, bitmask_expand_rows_ok), semi-structured
# ------------------------------------------------------------------------------------------------------------------------------
def _sparse_x(rows, cols, density, dtype=torch.bfloat16, seed=0):
    g = torch.Generator().manual_seed(seed + rows * 7 + cols)
    x = (torch.randn(rows, cols, generator=g) * 3).to(dtype)
    x[torch.rand(rows, cols, generator=g) >= density] = 0
    return x


BITMASK_SHAPES = [(1, 8, "one-unit"), (3, 13, "cols%8"), (5, 8 * 1023, "tile-1"), (2, 8 * 1024, "tile"), (1, 8 * 1025 * 4, "tile+1"),
                  (7, 8 * 3, "units%G"), (64, 128, "many-rows")]


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [256, 16, 2])
def test_bitmasks_and_24(offset):
    lib = N.lib()
    for rows, cols, what in BITMASK_SHAPES:
        m = (torch.rand(rows, cols, generator=torch.Generator().manual_seed(cols)) < 0.5).to(torch.uint8)
        pk = oracle.pack_bitmasks(m)
        run_fenced("ct_pack_bitmasks", f"{what}-{rows}x{cols}-off{offset}", {"m": m}, {"o": (tuple(pk.shape), torch.uint8)},
                   lambda i, o: lib.ct_pack_bitmasks(N.ptr(i["m"]), N.ptr(o["o"]), rows, cols, 0, _st()), {"o": pk},
                   offset=offset, device=DEV)
        run_fenced("ct_unpack_bitmasks", f"{what}-{rows}x{cols}-off{offset}", {"p": pk}, {"o": ((rows, cols), torch.uint8)},
                   lambda i, o: lib.ct_unpack_bitmasks(N.ptr(i["p"]), N.ptr(o["o"]), rows, cols, 0, _st()), {"o": m},
                   offset=offset, device=DEV)
        if cols % 4:
            continue
        x = _sparse_x(rows, cols, 1.0)
        vals, bm = oracle.sparse24_compress(x)
        path = ("vec16" if cols % 8 == 0 else "scalar") if offset >= 16 else "scalar-misaligned"
        run_fenced("ct_sparse24_compress", f"{path}-{what}-{rows}x{cols}-off{offset}", {"x": x},
                   {"v": (tuple(vals.shape), x.dtype), "b": (tuple(bm.shape), torch.uint8)},
                   lambda i, o: lib.ct_sparse24_compress(N.ptr(i["x"]), N.DT[x.dtype], N.ptr(o["v"]), N.ptr(o["b"]), rows, cols, 0, _st()),
                   {"v": vals, "b": bm}, offset=offset, device=DEV)
        run_fenced("ct_sparse24_decompress", f"{path}-{what}-{rows}x{cols}-off{offset}", {"v": vals, "b": bm},
                   {"o": ((rows, cols), x.dtype)},
                   lambda i, o: lib.ct_sparse24_decompress(N.ptr(i["v"]), N.DT[x.dtype], N.ptr(i["b"]), N.ptr(o["o"]), rows, cols, 0, _st()),
                   {"o": oracle.sparse24_decompress(vals, bm, (rows, cols))}, offset=offset, device=DEV)


@pytest.mark.gpu
@pytest.mark.parametrize("density", [0.0, 0.4, 1.0])
@pytest.mark.parametrize("offset", [256, 16, 2])
def test_bitmask_unstructured(density, offset):
    lib = N.lib()
    for rows, cols, what in BITMASK_SHAPES:
        x = _sparse_x(rows, cols, density, seed=int(density * 10))
        vals, bm, offs = oracle.bitmask_compress(x)
        nnz = vals.numel()
        lookback = (rows * cols) % 32 == 0 and cols % 8 == 0 and offset >= 16
        path = "lookback" if lookback else "twophase"
        case = f"{path}-{what}-{rows}x{cols}-d{density}-off{offset}"
        outs = {"v": ((rows * cols,), x.dtype), "b": (tuple(bm.shape), torch.uint8), "r": ((rows,), torch.int64), "n": ((1,), torch.int64)}
        # values: a buffer of capacity rows * cols of which the first nnz are defined
        run_fenced("ct_bitmask_compress_onepass", case, {"x": x}, outs,
                   lambda i, o: lib.ct_bitmask_compress_onepass(N.ptr(i["x"]), N.DT[x.dtype], N.ptr(o["v"]), N.ptr(o["b"]), N.ptr(o["r"]),
                                                                N.ptr(o["n"]), rows, cols, 0, _st()),
                   {"v": vals, "b": bm, "r": offs, "n": torch.tensor([nnz])}, offset=offset, device=DEV,
                   valid={"v": lambda o: int(o["n"].item())})
        ws = torch.empty(lib.ct_bitmask_workspace_bytes(rows, cols), dtype=torch.uint8, device=DEV)
        run_fenced("ct_bitmask_count", case, {"x": x},
                   {"b": (tuple(bm.shape), torch.uint8), "r": ((rows,), torch.int64), "n": ((1,), torch.int64)},
                   lambda i, o: lib.ct_bitmask_count(N.ptr(i["x"]), N.DT[x.dtype], N.ptr(o["b"]), N.ptr(o["r"]), N.ptr(o["n"]), N.ptr(ws),
                                                     rows, cols, 0, _st()),
                   {"b": bm, "r": offs, "n": torch.tensor([nnz])}, offset=offset, device=DEV)
        run_fenced("ct_bitmask_compress", case, {"x": x, "b": bm, "r": offs}, {"v": ((nnz,), x.dtype)},
                   lambda i, o: lib.ct_bitmask_compress(N.ptr(i["x"]), N.DT[x.dtype], N.ptr(i["b"]), N.ptr(i["r"]), N.ptr(o["v"]),
                                                        rows, cols, 0, _st()),
                   {"v": vals}, offset=offset, device=DEV)
        dense = oracle.bitmask_decompress(vals, bm, (rows, cols))
        for with_offsets in (True, False):
            if not with_offsets and not lookback:
                continue
            # without row_offsets the values are the compress's capacity buffer (rows * cols elements, the first nnz defined)
            v_in = vals if with_offsets else torch.cat([vals, torch.zeros(rows * cols - nnz, dtype=x.dtype)])
            run_fenced("ct_bitmask_decompress", case + ("" if with_offsets else "-no-row-offsets"), {"v": v_in, "b": bm, "r": offs},
                       {"o": ((rows, cols), x.dtype)},
                       lambda i, o: lib.ct_bitmask_decompress(N.ptr(i["v"]), N.DT[x.dtype], N.ptr(i["b"]),
                                                              N.ptr(i["r"]) if with_offsets else None, N.ptr(o["o"]), rows, cols, 0, _st()),
                       {"o": dense}, offset=offset, device=DEV)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32, torch.int8])
def test_semi_structured(dtype):
    lib = N.lib()
    for m, k in ((64, 64), (128, 192)):
        x = _sparse_x(m, k, 1.0).float()
        x = x.unflatten(-1, (-1, 4))
        x[..., 1] = 0
        x[..., 3] = 0
        dense = (x.flatten(-2) * (10 if dtype == torch.int8 else 1)).to(dtype)
        if dtype == torch.float32:
            dense = dense.unflatten(-1, (-1, 2)).clone()
            dense[..., 1] = 0
            dense = dense.flatten(-2)
        sp, meta = oracle.semi_structured_from_dense(dense)
        run_fenced("ct_semi_structured_from_dense", f"{m}x{k}-{str(dtype)[6:]}", {"d": dense},
                   {"s": (tuple(sp.shape), dtype), "m": (tuple(meta.shape), meta.dtype)},
                   lambda i, o: lib.ct_semi_structured_from_dense(N.ptr(i["d"]), N.DT[dtype], N.ptr(o["s"]), N.ptr(o["m"]), m, k, 0, _st()),
                   {"s": sp, "m": meta}, device=DEV)
        run_fenced("ct_semi_structured_to_dense", f"{m}x{k}-{str(dtype)[6:]}", {"s": sp, "m": meta}, {"d": ((m, k), dtype)},
                   lambda i, o: lib.ct_semi_structured_to_dense(N.ptr(i["s"]), N.DT[dtype], N.ptr(i["m"]), N.ptr(o["d"]), m, k // 2, 0, _st()),
                   {"d": oracle.semi_structured_to_dense(sp, meta)}, device=DEV)


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [256, 32, 16])
def test_sparse24_int4(offset):
    from types import SimpleNamespace as NS

    lib = N.lib()
    for rows, cols, group in ((2, 32, 32), (3, 128 * 5, 128), (6, 32 * 2049, 32), (2, 64 * 3, 64)):
        x = _x(rows, cols, seed=8)
        args = NS(strategy="group", group_size=group, num_bits=4, type="int")
        amax = x.float().unflatten(-1, (-1, group)).abs().amax(-1)
        scale = (amax / 7 + 2 ** -8).to(x.dtype)
        zp = torch.randint(-2, 3, scale.shape, dtype=torch.int8, generator=torch.Generator().manual_seed(cols))
        wp, wb = oracle.sparse24_quantize_pack(x, scale, zp, strategy="group", group_size=group)
        p = ops._resolve(x, scale, zp, args, None)
        d = ops._desc(p, x.dtype, scale.dtype, torch.int8, x.dtype, torch.int8, None, N.Q_INT, 4)
        run_fenced("ct_sparse24_quantize_pack_int4", f"fast-g{group}-{rows}x{cols}-off{offset}", {"x": x, "s": scale, "z": zp},
                   {"p": (tuple(wp.shape), torch.int32), "b": (tuple(wb.shape), torch.uint8)},
                   lambda i, o: lib.ct_sparse24_quantize_pack_int4(ctypes.byref(d), N.ptr(i["x"]), N.ptr(i["s"]), N.ptr(i["z"]),
                                                                   N.ptr(o["p"]), N.ptr(o["b"]), 0, _st()),
                   {"p": wp, "b": wb}, offset=offset, device=DEV)
        want = oracle.sparse24_unpack_dequantize(wp, wb, scale, zp, 4, (rows, cols))
        d2 = ops._desc(p, None, scale.dtype, torch.int8, None, torch.int8, x.dtype, N.Q_INT, 4)
        if offset % 32:
            # the expansion writes with 256-bit stores and has no other kernel: a 16-byte aligned output is declined, nothing written
            out, check = fenced((rows, cols), x.dtype, offset, POISONS[0], DEV, label="output o")
            rc = lib.ct_sparse24_unpack_dequantize_int4(ctypes.byref(d2), N.ptr(wp.to(DEV)), N.ptr(wb.to(DEV)), N.ptr(scale.to(DEV)),
                                                        N.ptr(zp.to(DEV)), N.ptr(out), 0, _st())
            assert rc == N.CT_E_UNSUPPORTED
            check()
            assert bool((out.view(torch.uint8) == POISONS[0]).all())
            continue
        path = "fast-256bit"
        run_fenced("ct_sparse24_unpack_dequantize_int4", f"{path}-g{group}-{rows}x{cols}-off{offset}",
                   {"p": wp, "b": wb, "s": scale, "z": zp}, {"o": ((rows, cols), x.dtype)},
                   lambda i, o: lib.ct_sparse24_unpack_dequantize_int4(ctypes.byref(d2), N.ptr(i["p"]), N.ptr(i["b"]), N.ptr(i["s"]),
                                                                       N.ptr(i["z"]), N.ptr(o["o"]), 0, _st()),
                   {"o": want.to(x.dtype)}, offset=offset, device=DEV)


# ------------------------------------------------------------------------------------------------------------------------------
# Walsh-Hadamard on the device, and K / V views cut from a fused qkv buffer
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("offset", [256, 16, 2])
def test_hadamard_transform(offset):
    from tests.test_transform_host import structured_reference

    for log2_n, shape in ((1, (1, 1, 1, 2)), (7, (2, 3, 5, 256)), (12, (1, 1, 3, 4096)), (15, (1, 1, 1, 32768))):
        n = 1 << log2_n
        g = torch.Generator().manual_seed(log2_n)
        x = torch.randn(shape, generator=g).bfloat16()
        sign = torch.where(torch.rand(n, generator=g) < 0.5, -1, 1).to(torch.int8)
        perm = torch.randperm(n, generator=g)
        want = structured_reference(x, n, sign, perm).float().bfloat16()

        def call(i, o):
            j = ops._hadamard_job(i["x"], o["o"], log2_n, i["sign"], i["perm"], False, torch.float64)
            return N.lib().ct_hadamard_transform(ctypes.byref(j), 0, _st())

        run_fenced("ct_hadamard_transform", f"n{n}-{'x'.join(map(str, shape))}-off{offset}", {"x": x, "sign": sign, "perm": perm},
                   {"o": (shape, torch.bfloat16)}, call, {"o": want}, offset=offset, device=DEV)


def _owned(shape, strides, offset_elems, total):
    """bool [total]: the elements of a flat buffer that the view (shape, strides, storage offset) covers"""
    idx = torch.arange(total).as_strided(shape, strides, offset_elems)
    m = torch.zeros(total, dtype=torch.bool)
    m[idx.reshape(-1)] = True
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_strided_kv_views(dtype):
    """K and V of a GQA model as the transposed [B, H, S, D] views of one fused qkv projection with padded rows: every element the
    views do not own -- Q, the padding, the other tensor -- keeps its value"""
    from types import SimpleNamespace as NS

    b, s, hq, hkv, d, pad = 2, 37, 8, 2, 64, 8
    row = (hq + 2 * hkv) * d + pad
    for run, poison in enumerate(POISONS):
        g = torch.Generator().manual_seed(run)
        src = (torch.randn(b * s * row, generator=g) * 2).to(dtype)
        fence = FencedInput("qkv", src, 256, in_guard(dtype, run), DEV)
        dst = Fence("qkv out", (b * s * row,), dtype, 256, bytes([poison]), DEV)
        qkv_in = fence.view.view(b, s, row)
        qkv_out = dst.view.view(b, s, row)
        views = []
        for t, start in (("k", hq * d), ("v", (hq + hkv) * d)):
            xi = qkv_in[..., start:start + hkv * d].unflatten(-1, (hkv, d)).transpose(1, 2)
            xo = qkv_out[..., start:start + hkv * d].unflatten(-1, (hkv, d)).transpose(1, 2)
            views.append((t, xi, xo))
        # fake-quantize both views in one launch
        args = NS(strategy="attn_head", num_bits=8, type="int", symmetric=False)
        jobs, keep, wants = (N.HeadJob * 2)(), [], []
        for k, (t, xi, xo) in enumerate(views):
            scale = (xi.float().abs().amax((0, 2, 3)) / 100 + 0.01).to(dtype).reshape(hkv, 1, 1).to(DEV)
            zp = torch.randint(-5, 6, (hkv, 1, 1), dtype=torch.int8, generator=g).to(DEV)
            wants.append(ops.fake_quantize(xi.contiguous(), scale, zp, args))
            j, _ = ops._head_job(xi, scale, zp, args, xo), keep.extend([scale, zp])
            jobs[k] = j[0] if isinstance(j, tuple) else j
        launches = N.launch_count()
        N.check(N.lib().ct_fake_quantize_heads(2, jobs, 0, _st()), "ct_fake_quantize_heads")
        assert N.launch_count() - launches == 1, "one launch for K and V"
        torch.cuda.synchronize()
        err = fence.changed()
        assert err is None, f"ct_fake_quantize_heads[gqa-padded run {run}]: {err}"
        owned = torch.zeros(b * s * row, dtype=torch.bool)
        for t, xi, xo in views:
            owned |= _owned(xo.shape, xo.stride(), xo.storage_offset() - dst.view.storage_offset(), b * s * row)
        out = dst.bytes().view(dtype)
        bad = (out.view(torch.uint8).view(-1, out.element_size()) != poison).any(1) & ~owned
        assert not bool(bad.any()), f"ct_fake_quantize_heads[gqa-padded run {run}]: element {int(bad.nonzero()[0])} not owned by K or V written"
        assert dst.guard_error() is None, f"ct_fake_quantize_heads[gqa-padded run {run}]: {dst.guard_error()}"
        for (t, xi, xo), want in zip(views, wants):
            got = xo.contiguous()
            assert torch.equal(got.view(torch.int16), want.view(torch.int16)), f"ct_fake_quantize_heads[{t}]: values differ"
        # the Walsh-Hadamard of the same views, in place of their strides
        for t, xi, xo in views:
            dst2 = Fence("qkv out", (b * s * row,), dtype, 256, bytes([poison]), DEV)
            start = hq * d if t == "k" else (hq + hkv) * d
            xo2 = dst2.view.view(b, s, row)[..., start:start + hkv * d]
            xo2 = xo2.unflatten(-1, (hkv, d)).transpose(1, 2)
            j = ops._hadamard_job(xi, xo2, 6, None, None, False, torch.float32)
            N.check(N.lib().ct_hadamard_transform(ctypes.byref(j), 0, _st()), "ct_hadamard_transform")
            torch.cuda.synchronize()
            assert fence.changed() is None, f"ct_hadamard_transform[gqa-{t} run {run}]: {fence.changed()}"
            mine = _owned(xo2.shape, xo2.stride(), xo2.storage_offset() - dst2.view.storage_offset(), b * s * row)
            out = dst2.bytes().view(dtype)
            bad = (out.view(torch.uint8).view(-1, out.element_size()) != poison).any(1) & ~mine
            assert not bool(bad.any()), f"ct_hadamard_transform[gqa-{t} run {run}]: element {int(bad.nonzero()[0])} outside the view written"
            assert dst2.guard_error() is None, f"ct_hadamard_transform[gqa-{t} run {run}]: {dst2.guard_error()}"
            want = ops.hadamard_transform(xi.contiguous(), 64)
            assert torch.equal(xo2.contiguous().view(torch.int16), want.view(torch.int16)), f"ct_hadamard_transform[gqa-{t}]: values differ"


# ------------------------------------------------------------------------------------------------------------------------------
# whole-model launches: 40+ tensors back to back in one fenced arena
# ------------------------------------------------------------------------------------------------------------------------------
class Arena:
    """tensors packed back to back at 16-byte aligned offsets in one fenced buffer; `check()` reports a write to any byte that
    belongs to none of them (the 16-byte gaps between them included)"""

    def __init__(self, label, specs, fill: bytes, device=DEV, values=None, pin=False, align=16):
        self.offs, off = [], 0
        for shape, dtype in specs:
            self.offs.append(off)
            off += math.prod(shape) * torch.empty((), dtype=dtype).element_size()
            off += -off % align
        self.f = Fence(label, (off,), torch.uint8, 256, fill, device, pin)
        self.views = []
        for (shape, dtype), o in zip(specs, self.offs):
            nb = math.prod(shape) * torch.empty((), dtype=dtype).element_size()
            v = self.f.view[o:o + nb].view(dtype).view(shape)
            self.views.append(v)
        if values is not None:
            for v, t in zip(self.views, values):
                v.copy_(t)
        self.owned = torch.zeros(off, dtype=torch.bool)
        for (shape, dtype), o in zip(specs, self.offs):
            self.owned[o:o + math.prod(shape) * torch.empty((), dtype=dtype).element_size()] = True
        self.snapshot = self.f.raw.clone()

    def error(self, inputs: bool):
        if inputs:
            bad = (self.f.raw != self.snapshot).nonzero()
            return None if bad.numel() == 0 else f"{self.f.label}: byte {int(bad[0]) - self.f.begin} of the arena written"
        e = self.f.guard_error()
        if e:
            return e
        body = self.f.view.cpu()
        k = len(self.f.fill)
        pat = torch.tensor(list(self.f.fill), dtype=torch.uint8).repeat(body.numel() // k + 1)[: body.numel()]
        bad = ((body != pat) & ~self.owned).nonzero()
        return None if bad.numel() == 0 else f"{self.f.label}: gap byte {int(bad[0])} between tensors written"


def _bproblem(op, i, seed):
    """(desc, in, scale, zp, per-tensor expected {out[, scale, zp]}) of tensor i of a batched op; shapes alternate fast and generic plans
    and sizes that are not multiples of 512 bytes"""
    from types import SimpleNamespace as NS

    rows = 1 + (i * 7) % 5
    cols = [8 * 37, 8 * 129, 40, 8 * 2049, 128 * 3, 13][i % 6]
    if op in ("PACK_INT32", "UNPACK_INT32"):
        bits = [4, 8, 3, 4, 8, 5][i % 6]
        codes = torch.randint(-(1 << (bits - 1)), 1 << (bits - 1), (rows, cols), dtype=torch.int8, generator=torch.Generator().manual_seed(seed + i))
        packed = oracle.pack_to_int32(codes, bits)
        d = N.QuantDesc()
        d.rows, d.cols, d.num_bits = rows, cols, bits
        if op == "PACK_INT32":
            return d, codes, None, None, {"out": packed}
        return d, packed, None, None, {"out": codes}
    if op in ("QUANTIZE_PACK", "UNPACK_DEQUANTIZE", "QUANTIZE", "DEQUANTIZE", "FAKE_QUANTIZE"):
        strategy, gs = [("group", 128), ("channel", None), ("tensor", None)][i % 3]
        if strategy == "group" and cols % 128:
            strategy, gs = "channel", None
        bits = 4 if op in ("QUANTIZE_PACK", "UNPACK_DEQUANTIZE") else 8
        x, scale, zp, args = qproblem(strategy, rows, cols, torch.bfloat16, bits, "int", asym=bool(i % 2), group_size=gs, seed=seed + i)
        name = {"QUANTIZE_PACK": "quantize_pack", "UNPACK_DEQUANTIZE": "unpack_dequantize", "QUANTIZE": "quantize",
                "DEQUANTIZE": "dequantize", "FAKE_QUANTIZE": "fake_quantize"}[op]
        d, want = quant_desc(name, x, scale, zp, args)
        ins, _ = quant_io(name, x, scale, zp, args, want)
        return d, ins["x"], ins["scale"], ins.get("zp"), {"out": want}
    x = _x(rows, cols if cols % 128 == 0 else 128 * (1 + i % 3), seed=seed + i)
    rows, cols = x.shape
    xd = x.to(DEV)
    if op == "OBSERVE_QUANTIZE_PACK":
        args = NS(strategy="group", group_size=128, num_bits=4, type="int", symmetric=False)
        p, s, z = ops.observe_quantize_pack(xd, args)
        d = N.QuantDesc()
        d.rows, d.cols, d.rdiv, d.cdiv, d.s_row_stride = rows, cols, 1, 128, cols // 128
        d.x_dtype = d.scale_dtype = d.compute_dtype = N.DT[x.dtype]
        d.zp_dtype, d.q_dtype, d.out_dtype, d.qtype, d.num_bits = N.DT[torch.int8], N.DT[torch.int8], N.DT_NONE, N.Q_INT, 4
        return d, x, ("out", s), ("out", z), {"out": p, "scale": s, "zp": z}
    if op == "OBSERVE_QUANTIZE_BLOCK":
        q, s = ops.observe_quantize(xd, NS(strategy="block", block_structure=[16, 128], num_bits=8, type="float", symmetric=True,
                                           group_size=None))[:2]
        return ops._block_desc(rows, cols, 16, 128, x.dtype), x, ("out", s.reshape(-1)), None, {"out": q, "scale": s.reshape(-1)}
    if op == "OBSERVE_QUANTIZE_MX":
        bits = 4 if i % 2 else 8
        q, s = ops.observe_quantize_mx(xd, NS(strategy="group", group_size=32, num_bits=bits, type="float", symmetric=True,
                                              scale_dtype=torch.uint8, block_structure=None))
        return ops._mx_desc(rows, cols, bits, x.dtype), x, ("out", s), None, {"out": q, "scale": s}
    if op == "QUANTIZE_PACK_FP4":
        scale = (x.float().unflatten(-1, (-1, 32)).abs().amax(-1) / 6 + 2 ** -8).to(x.dtype)
        args = NS(strategy="group", group_size=32, num_bits=4, type="float")
        want = ops.quantize_pack_fp4(xd, scale.to(DEV), None, args)
        p = ops._resolve(x, scale, None, args, None)
        return ops._desc(p, x.dtype, x.dtype, None, x.dtype, x.dtype, None, N.Q_FP4, 4, x.dtype), x, scale, None, {"out": want}
    if op == "UNPACK_DEQUANTIZE_FP4":
        scale = (x.float().unflatten(-1, (-1, 32)).abs().amax(-1) / 6 + 2 ** -8).to(x.dtype)
        args = NS(strategy="group", group_size=32, num_bits=4, type="float")
        packed = ops.quantize_pack_fp4(xd, scale.to(DEV), None, args)
        want = ops.unpack_dequantize_fp4(packed, scale.to(DEV), dtype=x.dtype)
        p = ops._resolve(x, scale, None, args, None)
        return ops._desc(p, None, x.dtype, None, None, None, x.dtype, N.Q_FP4, 4, x.dtype), packed.cpu(), scale, None, {"out": want}
    if op == "OBSERVE_QUANTIZE_PACK_FP4":
        args = NS(strategy="tensor_group", group_size=16, num_bits=4, type="float", symmetric=True)
        gsc = torch.tensor([448 * 6 / float(x.float().abs().max())], dtype=torch.float32)
        pk, s, _ = ops.observe_quantize_pack_nvfp4(xd, args, gsc.to(DEV))
        d = N.QuantDesc()
        d.rows, d.cols, d.rdiv, d.cdiv, d.s_row_stride = rows, cols, 1, 16, cols // 16
        d.x_dtype, d.scale_dtype, d.compute_dtype = N.DT[x.dtype], N.DT[torch.float8_e4m3fn], N.DT[torch.float32]
        d.zp_dtype, d.q_dtype, d.out_dtype, d.qtype, d.num_bits = N.DT_NONE, N.DT[x.dtype], N.DT_NONE, N.Q_FP4, 4
        d.seff_dtype = N.DT[torch.float32]
        return d, x, ("out", s), None, {"out": pk, "scale": s, "gs": gsc}
    # 2:4 + int4: descs[i].aux is the bitmask (an output of the compress, an input of the expansion).  The fused kernels take full rows
    # of scales only: a one-row weight (one shared scale row) is declined, so every weight here has two rows or more
    if rows == 1:
        x = torch.cat([x, x.flip(0) * 0.5])
        rows = 2
    scale = (x.float().unflatten(-1, (-1, 128)).abs().amax(-1) / 7 + 2 ** -8).to(x.dtype)
    wp, wb = oracle.sparse24_quantize_pack(x, scale, None, strategy="group", group_size=128)
    args = NS(strategy="group", group_size=128, num_bits=4, type="int")
    p = ops._resolve(x, scale, None, args, None)
    if op == "SPARSE24_QUANTIZE_PACK":
        d = ops._desc(p, x.dtype, x.dtype, None, x.dtype, torch.int8, None, N.Q_INT, 4)
        return d, x, scale, None, {"out": wp, "aux": wb}
    d = ops._desc(p, None, x.dtype, None, None, torch.int8, x.dtype, N.Q_INT, 4)
    want = oracle.sparse24_unpack_dequantize(wp, wb, scale, None, 4, (rows, cols)).to(x.dtype)
    return d, wp, scale, None, {"out": want, "aux_in": wb}


BATCH_OPS = ["QUANTIZE_PACK", "UNPACK_DEQUANTIZE", "QUANTIZE", "DEQUANTIZE", "FAKE_QUANTIZE", "PACK_INT32", "UNPACK_INT32",
             "OBSERVE_QUANTIZE_PACK", "QUANTIZE_PACK_FP4", "UNPACK_DEQUANTIZE_FP4", "OBSERVE_QUANTIZE_PACK_FP4", "SPARSE24_QUANTIZE_PACK",
             "SPARSE24_UNPACK_DEQUANTIZE", "OBSERVE_QUANTIZE_BLOCK", "OBSERVE_QUANTIZE_MX"]


def run_arena(op: str, n: int, seed: int, *, host: bool = False, pin: bool = False, graph: bool = False, problems=None):
    """every tensor of a batched op in fenced arenas (inputs, input scales / zero points, outputs, output scales / zero points, 2:4
    masks); both poisons; each output equals its own per-tensor expectation.  host: through ct_host_run_many on host buffers."""
    opnum = getattr(N, f"OP_{op}")
    problems = problems or [_bproblem(op, i, seed) for i in range(n)]
    device = "cpu" if host else DEV
    outs_spec = [(tuple(p[4]["out"].shape), p[4]["out"].dtype) for p in problems]
    for run, poison in enumerate(POISONS):
        ins = Arena("inputs", [(tuple(p[1].shape), p[1].dtype) for p in problems], in_guard(problems[0][1].dtype, run), device,
                    [p[1] for p in problems], pin)
        outs = Arena("outputs", outs_spec, bytes([poison]), device, None, pin, 32 if op.startswith("SPARSE24") else 16)
        side = {}
        for role, k in (("scale", 2), ("zp", 3)):
            items = [(i, p[k]) for i, p in enumerate(problems) if p[k] is not None]
            if not items:
                continue
            is_out = isinstance(items[0][1], tuple)
            tens = [t[1] if is_out else t for _, t in items]
            a = Arena(f"{'output' if is_out else 'input'} {role}", [(tuple(t.shape), t.dtype) for t in tens],
                      bytes([poison]) if is_out else in_guard(tens[0].dtype, run), device, None if is_out else tens, pin)
            side[role] = (a, dict(zip([i for i, _ in items], a.views)), is_out)
        aux = None
        if "aux" in problems[0][4] or "aux_in" in problems[0][4]:
            is_out = "aux" in problems[0][4]
            tens = [p[4]["aux" if is_out else "aux_in"] for p in problems]
            aux = Arena("output 2:4 masks" if is_out else "input 2:4 masks", [(tuple(t.shape), t.dtype) for t in tens],
                        bytes([poison]) if is_out else b"\x77", device, None if is_out else tens, pin)
        gsv = None
        if "gs" in problems[0][4]:
            gsv = [FencedInput("global scale", p[4]["gs"], 256, in_guard(torch.float32, run), device) for p in problems]
        descs = []
        for i, p in enumerate(problems):
            d = N.QuantDesc.from_buffer_copy(p[0])
            if aux is not None:
                d.aux = aux.views[i].data_ptr()
            if gsv is not None:
                d.global_scale = gsv[i].view.data_ptr()
            descs.append(d)
        table = [(descs[i], ins.views[i], side["scale"][1].get(i) if "scale" in side else None,
                  side["zp"][1].get(i) if "zp" in side else None, outs.views[i]) for i in range(len(problems))]
        dt, ip, sp, zp_, op_ = ops._tables(table)
        if "scale" not in side:
            sp = (ctypes.c_void_p * len(problems))()
        args = (opnum, len(problems), dt, ctypes.cast(ip, ctypes.c_void_p), ctypes.cast(sp, ctypes.c_void_p),
                ctypes.cast(zp_, ctypes.c_void_p), ctypes.cast(op_, ctypes.c_void_p))
        if host:
            rc = N.lib().ct_host_run_many(*args, 0)
        elif graph:
            s = torch.cuda.Stream()
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr, stream=s):
                rc = N.lib().ct_batched(*args, 0, ctypes.c_void_p(s.cuda_stream))
            assert rc == N.CT_OK, N.last_error()
            gr.replay()
        else:
            rc = N.lib().ct_batched(*args, 0, _st())
        if not host:
            torch.cuda.synchronize()
        where = f"{'ct_host_run_many' if host else 'ct_batched'}[{op} n={len(problems)}{' graph' if graph else ''} run {run}]"
        assert rc == N.CT_OK, f"{where}: status {rc}: {N.last_error()}"
        errs = [ins.error(True), outs.error(False)] + [a.error(not o) for a, _, o in side.values()]
        errs += [aux.error("aux_in" in problems[0][4])] if aux is not None else []
        errs += [g.changed() for g in gsv] if gsv else []
        errs = [e for e in errs if e]
        assert not errs, f"{where}: " + "; ".join(errs)
        for i, p in enumerate(problems):
            checks = [("out", outs.views[i])]
            if "scale" in side and side["scale"][2]:
                checks.append(("scale", side["scale"][1][i]))
            if "zp" in side and side["zp"][2]:
                checks.append(("zp", side["zp"][1][i]))
            if aux is not None and "aux" in p[4]:
                checks.append(("aux", aux.views[i]))
            for name, got in checks:
                want = p[4][name].to(got.device)
                from tests.test_write_fences_host import _nan_equal
                j = _nan_equal(got.reshape(-1).cpu(), want.reshape(-1).cpu())
                assert j is None, f"{where}: tensor {i} {name} element {j} differs from its per-tensor expectation"


@pytest.mark.gpu
@pytest.mark.parametrize("op", BATCH_OPS)
def test_batched_arena(op):
    run_arena(op, 41, seed=BATCH_OPS.index(op))


@pytest.mark.gpu
def test_batched_arena_dynamic_and_graph():
    # DYNAMIC_MIN_TILES_PER_SM (24) x 132 SMs x 1024-chunk tiles of 8 elements: 26M fake-quantized elements take the dynamic claim
    probs = []
    for i in range(41):
        x, scale, zp, args = qproblem("channel", 160 + i % 3, 4096 + 8 * (i % 5), torch.bfloat16, 8, "int", asym=bool(i % 2), seed=i)
        d, want = quant_desc("fake_quantize", x, scale, zp, args)
        probs.append((d, x, scale.contiguous(), zp.contiguous() if zp is not None else None, {"out": want}))
    big = []
    for i in range(41):
        x, scale, zp, args = qproblem("tensor", 640, 1000 + 8 * i, torch.bfloat16, 8, "int", asym=False, seed=100 + i)
        d, want = quant_desc("fake_quantize", x, scale, zp, args)
        big.append((d, x, scale.contiguous(), None, {"out": want}))
    assert sum(p[1].numel() for p in big) >= 24 * 132 * 1024 * 8
    run_arena("FAKE_QUANTIZE", len(big), 0, problems=big)
    run_arena("FAKE_QUANTIZE", len(probs), 0, problems=probs, graph=True)


@pytest.mark.gpu
@pytest.mark.parametrize("pin", [True, False], ids=["pinned", "pageable"])
@pytest.mark.parametrize("op", ["QUANTIZE_PACK", "UNPACK_DEQUANTIZE", "FAKE_QUANTIZE", "DEQUANTIZE", "QUANTIZE"])
def test_host_run_many(op, pin, monkeypatch):
    monkeypatch.setenv("CT_B200_HOST_CHUNK_MB", "1")     # 1 MiB chunks: tensors span chunks and the last one is partial
    probs = [_bproblem(op, i, 50) for i in range(40)]
    run_arena(op, 40, 50, host=True, pin=pin, problems=probs)
