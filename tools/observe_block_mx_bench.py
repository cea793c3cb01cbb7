#!/usr/bin/env python
"""
Calibrate-and-compress of the full Llama-3-8B weight set (32 layers, 224 bf16 weights, 13.96 GB) in the FP8_BLOCK, MXFP4 and MXFP8
formats, three ways:
    batched    one ct_batched launch of CT_OP_OBSERVE_QUANTIZE_BLOCK / _MX over every weight (ops.BatchedPlan.run)
    per-tensor ops.observe_quantize (BLOCK) / ops.observe_quantize_mx, one call per weight
    unfused    torch min / max per block or group -> calculate_qparams -> ops.quantize / ops.quantize_pack_fp4 (-> ops.compress_mx_scale)
Times are CUDA events around `iters` whole-model passes after `warmup` passes; GB/s counts the bytes the format needs (weight read once,
codes and scales written once).  The copy rate of tools/hbm_ceilings.py's kernel, the card, its power limit and max SM clock are
measured in the same run, and every weight's fused output is checked bit for bit against the unfused one.

    python tools/observe_block_mx_bench.py [--iters 5] [--warmup 2] [--json out.json]
"""
import argparse
import json
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from compressed_tensors_b200 import _native as N  # noqa: E402
from compressed_tensors_b200 import ops  # noqa: E402
from compressed_tensors_b200.quantization import calculate_qparams, preset_name_to_scheme  # noqa: E402
from tools.dynamic_quant_bench import card, time_call  # noqa: E402
from tools.hbm_ceilings import rate  # noqa: E402

F8 = torch.float8_e4m3fn


def unfused(fmt, w, args):
    if fmt == "FP8_BLOCK":
        bh, bw = args.block_structure
        r, c = w.shape
        nrb, ncb = math.ceil(r / bh), math.ceil(c / bw)
        wp = torch.nn.functional.pad(w, (0, ncb * bw - c, 0, nrb * bh - r)).reshape(nrb, bh, ncb, bw)
        s, _ = calculate_qparams(wp.amin(dim=(1, 3)), wp.amax(dim=(1, 3)), args)
        return ops.quantize(w, s, None, args, dtype=F8), s
    g = w.unflatten(-1, (-1, 32))
    s, _ = calculate_qparams(g.amin(-1), g.amax(-1), args)
    q = ops.quantize_pack_fp4(w, s, None, args) if args.num_bits == 4 else ops.quantize(w, s, None, args, dtype=F8)
    return q, ops.compress_mx_scale(s, torch.uint8)


def fused(fmt, w, args):
    if fmt == "FP8_BLOCK":
        q, s, _ = ops.observe_quantize(w, args)
        return q, s
    return ops.observe_quantize_mx(w, args)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("observe_block_mx_bench needs a CUDA device")
    name, power = card()
    n = 1 << 30
    src, dst = torch.ones(n, dtype=torch.bfloat16, device="cuda"), torch.empty(n, dtype=torch.bfloat16, device="cuda")
    copy_gbps = rate(lambda: dst.copy_(src), n * 4)
    del src, dst
    torch.cuda.empty_cache()
    print(f"device: {name}; power.limit, clocks.max.sm: {power}; copy rate (tools/hbm_ceilings.py kernel): {copy_gbps:.0f} GB/s")

    ws, _ = bench.make_weights(torch.device("cuda", 0), a.layers, 1000)
    numel = sum(w.numel() for w in ws)
    print(f"{len(ws)} weights, {numel * 2 / 1e9:.2f} GB bf16")
    results = {}
    for fmt in ("FP8_BLOCK", "MXFP4", "MXFP8"):
        args = preset_name_to_scheme(fmt, ["Linear"]).weights
        problems, nbytes = [], 0
        for w in ws:
            r, c = w.shape
            if fmt == "FP8_BLOCK":
                d = ops._block_desc(r, c, 128, 128, w.dtype)
                s = torch.empty((math.ceil(r / 128), math.ceil(c / 128)), dtype=w.dtype, device=w.device)
                q = torch.empty((r, c), dtype=F8, device=w.device)
            else:
                d = ops._mx_desc(r, c, args.num_bits, w.dtype)
                s = torch.empty((r, c // 32), dtype=torch.uint8, device=w.device)
                q = torch.empty((r, c // 2) if args.num_bits == 4 else (r, c), dtype=torch.uint8 if args.num_bits == 4 else F8, device=w.device)
            problems.append((d, w, s, None, q))
            nbytes += w.numel() * 2 + q.numel() * q.element_size() + s.numel() * s.element_size()
        op = N.OP_OBSERVE_QUANTIZE_BLOCK if fmt == "FP8_BLOCK" else N.OP_OBSERVE_QUANTIZE_MX
        plan = ops.BatchedPlan(op, problems)
        # bit identity of every weight: batched == per-tensor == unfused
        plan.run()
        mism = 0
        for (_, w, s, _, q) in problems:
            fq, fs = fused(fmt, w, args)
            uq, us = unfused(fmt, w, args)
            for x, y in ((q, fq), (q, uq), (s, fs), (s, us)):
                mism += int(not torch.equal(x.view(torch.uint8), y.view(torch.uint8)))
            del fq, fs, uq, us
        torch.cuda.empty_cache()
        row = {"bytes": nbytes, "mismatching_tensors": mism}
        for how, fn in (("batched", plan.run), ("per_tensor", lambda: [fused(fmt, w, args) for w in ws]),
                        ("unfused", lambda: [unfused(fmt, w, args) for w in ws])):
            us = time_call(fn, a.iters, a.warmup)
            row[how] = {"ms": round(us / 1e3, 3), "GB/s": round(nbytes / (us * 1e-6) / 1e9, 1),
                        "of_copy": round(nbytes / (us * 1e-6) / 1e9 / copy_gbps, 3)}
            torch.cuda.empty_cache()
        results[fmt] = row
        print(fmt, json.dumps(row))
        del plan, problems
        torch.cuda.empty_cache()
    out = dict(device=name, power=power, copy_gbps=copy_gbps, iters=a.iters, warmup=a.warmup, weights=len(ws), results=results)
    print(json.dumps(out))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
