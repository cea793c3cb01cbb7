#!/usr/bin/env python
"""
Per-launch timing distribution of the multi-tensor ops on one H100 (one CUDA-event pair per launch):
tells a systematic slowdown from sporadic stalls.  Prints one JSON line per op.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import headline_problems  # noqa: E402
from compressed_tensors_b200 import _native as N  # noqa: E402
from compressed_tensors_b200 import ops  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=8)
    ap.add_argument("--launches", type=int, default=40)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    P, OPS, n = headline_problems.build_problems(a.layers)
    codes = [torch.randint(-8, 8, (14336, 4096), dtype=torch.int8, device=dev) for _ in range(16)]
    pk = [torch.empty(c.shape[0], c.shape[1] // 8, dtype=torch.int32, device=dev) for c in codes]
    descs = []
    for c in codes:
        d = N.QuantDesc()
        d.rows, d.cols, d.num_bits = c.shape[0], c.shape[1], 4
        descs.append(d)
    nel = sum(c.numel() for c in codes)
    jobs = {k: (op, P[k], n * bpe) for k, (op, bpe) in OPS.items()}
    jobs["int4_pack"] = (N.OP_PACK_INT32, [(d, c, None, None, o) for d, c, o in zip(descs, codes, pk)], nel * 1.5)
    jobs["int4_unpack"] = (N.OP_UNPACK_INT32, [(d, o, None, None, c) for d, c, o in zip(descs, codes, pk)], nel * 1.5)
    # checkpoint converters: FP8 128x128-block dequantize (DeepSeek-style shapes) and the AutoAWQ nibble transpose
    fw = [torch.randn(7168, 4096, device=dev).to(torch.float8_e4m3fn) for _ in range(8)]
    fs = [torch.rand(56, 32, device=dev) * 0.01 + 1e-4 for _ in fw]
    fo = [torch.empty(w.shape, dtype=torch.bfloat16, device=dev) for w in fw]
    fprobs = [(ops._dequantize_block_fp8_call(w, sc, (128, 128)).desc, w, sc, None, o) for w, sc, o in zip(fw, fs, fo)]
    jobs["fp8_block_dq"] = (N.OP_DEQUANTIZE, fprobs, sum(w.numel() for w in fw) * 3.0)
    awq_q = torch.randint(-2 ** 31, 2 ** 31 - 1, (14336, 4096 // 8), device=dev, dtype=torch.int64).to(torch.int32)
    extra_fns = {"awq_repack": (lambda: ops.awq_repack(awq_q), 14336 * 4096 * 1.0)}
    # sparse formats (north-star rows a12 / a13): 2:4 bitmask and unstructured bitmask on one big bf16 tensor
    sp = (torch.randn(14336, 8192, device=dev) * 0.02).to(torch.bfloat16)
    nsp = sp.numel()
    vals24, mask24 = ops.sparse24_compress(sp)
    extra_fns["sparse24_compress"] = (lambda: ops.sparse24_compress(sp), nsp * 3.125)
    extra_fns["sparse24_decompress"] = (lambda: ops.sparse24_decompress(vals24, mask24, sp.shape), nsp * 3.125)
    from compressed_tensors_b200.quantization import QuantizationArgs
    for nm, kw, pk, bpe in (("observe_channel_int8", dict(num_bits=8, type="int"), False, 3.0), ("observe_channel_fp8", dict(num_bits=8, type="float"), False, 3.0),
                            ("observe_channel_w4pack", dict(num_bits=4, type="int"), True, 2.5)):
        qa_c = QuantizationArgs(strategy="channel", symmetric=True, **kw)
        extra_fns[nm] = ((lambda qa_c=qa_c, pk=pk: ops.observe_quantize(sp, qa_c, pack=pk)), nsp * bpe)
    un = torch.where(torch.rand(sp.shape, device=dev) < 0.5, sp, torch.zeros_like(sp))
    uv, um, uo = ops.bitmask_compress(un)
    extra_fns["bitmask_compress_50pct"] = (lambda: ops.bitmask_compress(un), nsp * (2 + 1 + 0.125))
    extra_fns["bitmask_decompress_50pct"] = (lambda: ops.bitmask_decompress(uv, um, uo, un.shape), nsp * (1 + 0.125 + 2))
    for name, (op, probs, nbytes) in jobs.items():
        for _ in range(3):
            ops.batched(op, probs, 0)
        torch.cuda.synchronize()
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(a.launches)]
        for e0, e1 in ev:
            e0.record()
            ops.batched(op, probs, 0)
            e1.record()
        torch.cuda.synchronize()
        ms = [e0.elapsed_time(e1) for e0, e1 in ev]
        s = sorted(ms)
        print(json.dumps({"op": name, "GBps_best": round(nbytes / s[0] / 1e6, 1),
                          "GBps_median": round(nbytes / s[len(s) // 2] / 1e6, 1), "GBps_worst": round(nbytes / s[-1] / 1e6, 1),
                          "ms": [round(v, 3) for v in ms]}), flush=True)
    # plain grid launches: their times include the output allocation
    for name, (fn, nbytes) in extra_fns.items():
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(a.launches)]
        for e0, e1 in ev:
            e0.record()
            fn()
            e1.record()
        torch.cuda.synchronize()
        s = sorted(e0.elapsed_time(e1) for e0, e1 in ev)
        print(json.dumps({"op": name, "GBps_best": round(nbytes / s[0] / 1e6, 1),
                          "GBps_median": round(nbytes / s[len(s) // 2] / 1e6, 1)}), flush=True)


if __name__ == "__main__":
    main()
