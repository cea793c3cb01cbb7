#!/usr/bin/env python
"""Per-launch medians (CUDA events) of the sparse-format kernels on one [14336, 8192] bf16 tensor (235 MB >> the 50 MB L2):
unstructured bitmask one-pass (look-back) vs two-phase, its expansion, 2:4 bitmask, and the fused 2:4 + int4 compressor of
BASELINE config 4.  Prints one JSON line per op; fractions are against the H100 SXM data-sheet HBM3 bandwidth, not a measured one.
The two-phase compression and the expansion without row_offsets are timed through their C ABI calls."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from compressed_tensors_b200 import _native as N, ops  # noqa: E402

dev = torch.device("cuda", 0)
torch.manual_seed(0)
PEAK = 3350.0   # GB/s: H100 SXM data sheet (HBM3, 3.35 TB/s)
lib, st = N.lib(), N.stream_ptr(0)
R, C = 14336, 8192
sp = (torch.randn(R, C, device=dev) * 0.02).to(torch.bfloat16)
n = sp.numel()


def med(fn, reps=21):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return sorted(a.elapsed_time(b) for a, b in ev)[reps // 2]


def report(name, ms, bytes_alg, **kw):
    gbs = bytes_alg / ms / 1e6
    print(json.dumps({"op": name, "us": round(ms * 1e3, 1), "alg_GBps": round(gbs, 1), "frac_of_datasheet_bw": round(gbs / PEAK, 3),
                      "alg_bytes_per_elem": round(bytes_alg / n, 4), **kw}), flush=True)


def bitmask_compress_two_phase(x):
    """count -> scan -> move into a values buffer of capacity numel, without a host synchronisation: what
    ct_bitmask_compress_onepass runs for the shapes its one-pass kernel declines"""
    rows, cols = x.shape
    bm = torch.empty((rows, (cols + 7) // 8), dtype=torch.uint8, device=dev)
    offs = torch.empty(rows, dtype=torch.int64, device=dev)
    nnz = torch.empty(1, dtype=torch.int64, device=dev)
    vals = torch.empty(x.numel(), dtype=x.dtype, device=dev)
    ws = torch.empty(lib.ct_bitmask_workspace_bytes(rows, cols), dtype=torch.uint8, device=dev)
    N.check(lib.ct_bitmask_count(N.ptr(x), N.DT[x.dtype], N.ptr(bm), N.ptr(offs), N.ptr(nnz), N.ptr(ws), rows, cols, 0, st))
    N.check(lib.ct_bitmask_compress(N.ptr(x), N.DT[x.dtype], N.ptr(bm), N.ptr(offs), N.ptr(vals), rows, cols, 0, st))


def bitmask_expand_no_row_offsets(vals, mask, shape):
    """the expansion without row_offsets: the look-back kernel recomputes the scan from the mask popcounts"""
    out = torch.empty(shape, dtype=vals.dtype, device=dev)
    N.check(lib.ct_bitmask_decompress(N.ptr(vals), N.DT[vals.dtype], N.ptr(mask), N.ptr(None), N.ptr(out), shape[0], shape[1], 0, st))


for density in (0.5, 0.1):
    un = torch.where(torch.rand(sp.shape, device=dev) < density, sp, torch.zeros_like(sp))
    vals, mask, offs = ops.bitmask_compress(un)
    d = vals.numel() / n
    b_alg = n * (2 + 2 * d + 0.125)
    report("bitmask_compress_onepass", med(lambda: ops.bitmask_compress(un, exact=False)), b_alg, density=round(d, 3))
    report("bitmask_expand_row_offsets", med(lambda: ops.bitmask_decompress(vals, mask, offs, un.shape)), b_alg, density=round(d, 3))
    report("bitmask_expand_lookback", med(lambda: bitmask_expand_no_row_offsets(vals, mask, un.shape)), b_alg, density=round(d, 3))
    report("bitmask_compress_two_phase", med(lambda: bitmask_compress_two_phase(un)), b_alg, density=round(d, 3))
    del un, vals, mask, offs

v24, m24 = ops.sparse24_compress(sp)
report("sparse24_compress", med(lambda: ops.sparse24_compress(sp)), n * 3.125)
report("sparse24_decompress", med(lambda: ops.sparse24_decompress(v24, m24, sp.shape)), n * 3.125)

if hasattr(ops, "sparse24_quantize_pack"):
    from types import SimpleNamespace

    from compressed_tensors_b200.utils.semi_structured_conversions import mask_creator

    w24 = sp * mask_creator(sp).to(sp.dtype)
    a = SimpleNamespace(strategy="group", group_size=128, block_structure=None, num_bits=4, type="int", symmetric=True)
    sc = (w24.unflatten(-1, (-1, 128)).abs().amax(-1).float() / 7.5).bfloat16()
    packed, bm = ops.sparse24_quantize_pack(w24, sc, None, a)
    report("sparse24_int4_compress", med(lambda: ops.sparse24_quantize_pack(w24, sc, None, a)), n * (2 + 0.25 + 0.125 + 2 / 128))
    report("sparse24_int4_decompress", med(lambda: ops.sparse24_unpack_dequantize(packed, bm, sc, None, 4, w24.shape)), n * (2 + 0.25 + 0.125 + 2 / 128))
