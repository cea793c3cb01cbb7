#!/usr/bin/env python
"""
KV-cache fake quantization on the H100: the one-launch strided op (ops.fake_quantize_heads) against the two-call path it replaces
(forward_quantize of K, then of V: a contiguous copy and a fake_quantize kernel each), on Llama-3-8B attention shapes.

    python tools/kv_quant_bench.py [--iters 200] [--warmup 20] [--json out.json]

K and V are [B, 8, S, 128] bf16 in the layout transformers hands to the KV-cache hook (the transpose of [B, S, 8, 128]), FP8 per-tensor
scales, 32 layers per timed step (one K / V pair per layer, each with its own tensors).  Per shape it prints the time per call (one K / V
pair) of the launch alone (prebuilt job tables), of both paths from CUDA events after warm-up, the algorithmic bandwidth (read + write of K and V, 4 bytes per element) and its share
of the H100 SXM's 3.35 TB/s, and checks in the same run that the two paths' outputs are bit-identical.  The card and its power limit are
printed with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from compressed_tensors_b200 import _native as N  # noqa: E402
from compressed_tensors_b200 import ops  # noqa: E402
from compressed_tensors_b200.quantization import QuantizationArgs  # noqa: E402
from compressed_tensors_b200.quantization.lifecycle.forward import forward_quantize  # noqa: E402

HBM_PEAK = 3.35e12
LAYERS = 32
SHAPES = {"prefill B=1 S=8192": (1, 8192), "prefill B=8 S=2048": (8, 2048), "decode B=64 S=1": (64, 1)}
KV_HEADS, HEAD_DIM = 8, 128


def card():
    name = torch.cuda.get_device_name()
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                               text=True, timeout=30).stdout.strip().splitlines()[torch.cuda.current_device()]
    except Exception as e:  # noqa: BLE001 -- report, do not guess
        power = f"unknown ({e})"
    return name, power


def layer_modules(args, gen):
    mods = []
    for _ in range(LAYERS):
        m = torch.nn.Module()
        for base in ("k", "v"):
            m.register_buffer(f"{base}_scale", (torch.rand(1, generator=gen) * 0.01 + 0.005).to(torch.bfloat16).cuda())
        mods.append(m)
    return mods


def time_path(fn, items, iters, warmup):
    for _ in range(warmup):
        for it in items:
            fn(*it)
    torch.cuda.synchronize()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        for it in items:
            fn(*it)
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) * 1e3 / (iters * len(items))   # us per K / V pair


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("kv_quant_bench needs a CUDA device")
    name, power = card()
    print(f"device: {name}; power.limit, clocks.max.sm: {power}")
    args = QuantizationArgs(num_bits=8, type="float", symmetric=True, strategy="tensor", dynamic=False)
    gen = torch.Generator().manual_seed(0)
    mods = layer_modules(args, gen)
    results = []
    for label, (b, s) in SHAPES.items():
        items = []
        for m in mods:
            k = torch.randn(b, s, KV_HEADS, HEAD_DIM, device="cuda", dtype=torch.bfloat16).transpose(1, 2)
            v = torch.randn(b, s, KV_HEADS, HEAD_DIM, device="cuda", dtype=torch.bfloat16).transpose(1, 2)
            items.append((m, k, v))

        def fused(m, k, v):
            return ops.fake_quantize_heads([k, v], [m.k_scale, m.v_scale], [None, None], args)

        def two_calls(m, k, v):
            return forward_quantize(m, k, "k", args), forward_quantize(m, v, "v", args)

        identical = True
        for m, k, v in items[:4]:
            for x, y in zip(fused(m, k, v), two_calls(m, k, v)):
                identical &= bool(torch.equal(x.contiguous().view(torch.int16), y.contiguous().view(torch.int16)))
        # the launch alone, job tables built once: what the kernel costs when the host keeps up (the Python layer above costs
        # ~30 us per call, more than the kernel at these sizes)
        lib, idx = N.lib(), torch.cuda.current_device()
        stream = N.stream_ptr(idx)
        tables = []
        for m, k, v in items:
            outs = (torch.empty_like(k), torch.empty_like(v))
            jobs = [ops._head_job(x, s, None, args, o) for x, s, o in ((k, m.k_scale, outs[0]), (v, m.v_scale, outs[1]))]
            tables.append(((N.HeadJob * 2)(*(j for j, _ in jobs)), (outs, jobs)))

        def launch_only(table, _outs):
            N.check(lib.ct_fake_quantize_heads(2, table, idx, stream), "ct_fake_quantize_heads")

        t_kernel = time_path(launch_only, tables, a.iters, a.warmup)
        t_fused = time_path(fused, items, a.iters, a.warmup)
        t_two = time_path(two_calls, items, a.iters, a.warmup)
        nbytes = 2 * 2 * b * s * KV_HEADS * HEAD_DIM * 2   # K and V, read + write, bf16
        row = dict(shape=label, B=b, S=s, us_launch_only=t_kernel, gbps_launch_only=nbytes / t_kernel / 1e3,
                   hbm_fraction_launch_only=nbytes / (t_kernel * 1e-6) / HBM_PEAK, us_fused=t_fused, us_two_calls=t_two, speedup=t_two / t_fused,
                   gbps_fused=nbytes / t_fused / 1e3, gbps_two_calls=nbytes / t_two / 1e3,
                   hbm_fraction_fused=nbytes / (t_fused * 1e-6) / HBM_PEAK, bit_identical=identical)
        results.append(row)
        print(f"{label:>20}: launch only {t_kernel:8.2f} us  {row['gbps_launch_only']:7.0f} GB/s "
              f"({row['hbm_fraction_launch_only']:.2f} of 3.35 TB/s) | fused {t_fused:8.2f} us  {row['gbps_fused']:7.0f} GB/s ({row['hbm_fraction_fused']:.2f} of 3.35 TB/s) | "
              f"two calls {t_two:8.2f} us  {row['gbps_two_calls']:7.0f} GB/s | x{row['speedup']:.2f} | bit-identical: {identical}")
    out = dict(device=name, power=power, layers=LAYERS, iters=a.iters, warmup=a.warmup, results=results)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=2)
    if not all(r["bit_identical"] for r in results):
        raise SystemExit("the fused and the two-call paths differ")


if __name__ == "__main__":
    main()
