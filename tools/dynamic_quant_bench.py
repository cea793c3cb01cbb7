#!/usr/bin/env python
"""
Dynamic activation fake quantization on the H100: the one-pass fused op (ops.dynamic_fake_quantize, the path forward_quantize takes)
against the two steps it replaces (compute_dynamic_scales_and_zp, then fake_quantize), for the input activations of FP8_DYNAMIC, W8A8,
FP8_BLOCK, NVFP4 and MXFP4 on Llama-3 activation shapes.

    python tools/dynamic_quant_bench.py [--iters 100] [--warmup 10] [--json out.json]

Per (shape, scheme) it prints the time per call from CUDA events after warm-up, three ways: the launch alone (ct_dynamic_fake_quantize
with prebuilt descriptor and outputs), forward_quantize on the fused path, and forward_quantize on the two-step path.  Algorithmic bytes
are one read and one write of the activation plus the scales and zero points written; the rate is given as a share of the H100 SXM's
3.35 TB/s data sheet and of the copy rate of tools/hbm_ceilings.py measured in the same run.  The two paths' outputs are checked for
bit-identity in the same run.  The card, its power limit and max SM clock are printed with the numbers.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from compressed_tensors_b200 import _native as N  # noqa: E402
from compressed_tensors_b200 import ops  # noqa: E402
from compressed_tensors_b200.quantization import preset_name_to_scheme  # noqa: E402
from compressed_tensors_b200.quantization.lifecycle.forward import forward_quantize  # noqa: E402
from tools.hbm_ceilings import rate  # noqa: E402

HBM_PEAK = 3.35e12
# Llama-3-8B prefill (attention / MLP input and the down-projection input), decode, and the Llama-3-70B down-projection
SHAPES = {"8B prefill [1, 8192, 4096]": (1, 8192, 4096), "8B prefill [1, 8192, 14336]": (1, 8192, 14336),
          "decode [64, 1, 4096]": (64, 1, 4096), "70B down [1, 4096, 28672]": (1, 4096, 28672)}
SCHEMES = ("FP8_DYNAMIC", "W8A8", "FP8_BLOCK", "NVFP4", "MXFP4")


def card():
    name = torch.cuda.get_device_name()
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                               text=True, timeout=30).stdout.strip().splitlines()[torch.cuda.current_device()]
    except Exception as e:  # noqa: BLE001 -- report, do not guess
        power = f"unknown ({e})"
    return name, power


def time_call(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) * 1e3 / iters   # us per call


def launch_only(x, args, gs):
    """the native call alone, descriptor and outputs built once (what ops.dynamic_fake_quantize enqueues)"""
    lib, idx = N.lib(), x.get_device()
    stream = N.stream_ptr(idx)
    captured = {}
    real = lib.ct_dynamic_fake_quantize

    class Rec:
        def ct_dynamic_fake_quantize(self, *a):
            captured["a"] = a
            return real(*a)

    orig = N.lib
    N.lib = lambda: Rec()
    try:
        keep = ops.dynamic_fake_quantize(x, args, global_scale=gs)
    finally:
        N.lib = orig
    a = captured["a"]
    desc = a[0]._obj   # the QuantDesc behind ctypes.byref

    def call():
        N.check(real(ctypes.byref(desc), *a[1:7], idx, stream), "ct_dynamic_fake_quantize")
    return call, keep


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dynamic_quant_bench needs a CUDA device")
    name, power = card()
    n = 1 << 30
    src, dst = torch.ones(n, dtype=torch.bfloat16, device="cuda"), torch.empty(n, dtype=torch.bfloat16, device="cuda")
    copy_gbps = rate(lambda: dst.copy_(src), n * 4)
    del src, dst
    print(f"device: {name}; power.limit, clocks.max.sm: {power}; copy rate (tools/hbm_ceilings.py kernel): {copy_gbps:.0f} GB/s")
    gen = torch.Generator(device="cuda").manual_seed(0)
    results = []
    for label, shape in SHAPES.items():
        x = torch.randn(shape, device="cuda", generator=gen).mul_(2).to(torch.bfloat16)
        for scheme in SCHEMES:
            args = preset_name_to_scheme(scheme, ["Linear"]).input_activations
            m = torch.nn.Module()
            gs = None
            if scheme == "NVFP4":
                gs = ops.observe_tensor_gparam(x)
                m.input_global_scale = gs
            kernel, (out, scale, zp) = launch_only(x, args, gs)
            real = ops.dynamic_fake_quantize

            def fused():
                return forward_quantize(m, x, "input", args)

            def two_step():
                ops.dynamic_fake_quantize = lambda *k, **kw: None
                try:
                    return forward_quantize(m, x, "input", args)
                finally:
                    ops.dynamic_fake_quantize = real

            identical = bool(torch.equal(fused().view(torch.int16), two_step().view(torch.int16)))
            t_kernel = time_call(kernel, a.iters, a.warmup)
            t_fused = time_call(fused, a.iters, a.warmup)
            t_two = time_call(two_step, a.iters, a.warmup)
            nbytes = 2 * x.numel() * x.element_size() + scale.numel() * scale.element_size() + zp.numel() * zp.element_size()
            gbps = nbytes / t_kernel / 1e3
            row = dict(shape=label, scheme=scheme, us_launch_only=t_kernel, gbps_launch_only=gbps, datasheet_fraction=gbps * 1e9 / HBM_PEAK,
                       copy_fraction=gbps / copy_gbps, us_fused=t_fused, us_two_step=t_two, two_step_over_fused=t_two / t_fused,
                       bit_identical=identical)
            results.append(row)
            print(f"{label:>28} {scheme:>11}: launch {t_kernel:8.1f} us {gbps:6.0f} GB/s ({row['datasheet_fraction']:.2f} of 3.35 TB/s, "
                  f"{row['copy_fraction']:.2f} of copy) | fused {t_fused:8.1f} us | two-step {t_two:8.1f} us | x{row['two_step_over_fused']:.1f} | "
                  f"bit-identical: {identical}")
        del x
    out = dict(device=name, power=power, copy_gbps=copy_gbps, iters=a.iters, warmup=a.warmup, results=results)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=2)
    if not all(r["bit_identical"] for r in results):
        raise SystemExit("the fused and the two-step paths differ")


if __name__ == "__main__":
    main()
