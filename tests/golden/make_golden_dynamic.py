#!/usr/bin/env python
"""
Golden vectors for dynamic activation quantization: the reference's compute_dynamic_scales_and_zp and forward_quantize (the dynamic
branch every quantized Linear's input takes) on seeded activations, by importing the reference exactly like make_golden.py does.

    python tests/golden/make_golden_dynamic.py   ->  tests/golden/dynamic.pt.gz

Schemes: the input activations of FP8_DYNAMIC, W8A8, W4A8, W4AFP8, FP8_BLOCK, NVFP4, MXFP4 and MXFP8, plus int8 per-token asymmetric
and int8 per-tensor asymmetric.  Inputs (bf16 and fp16, 2-D / 3-D / 4-D, rows up to 32768 wide, row and group counts that are not a
multiple of any tile) are randn with 1 % outliers at 50x; 2-D views with at least 4 rows also get an all-zero row (the eps scale), a row
of subnormal values (for fp16 MX groups the power-of-two scale underflows to 0 and becomes 1), a row of fp4 rounding ties under a unit
scale and a row of fp8 ties under a unit scale, both with -0.0.  NVFP4 runs with a global scale of 1 (the ties stay ties) and with
generate_gparam of the input.
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg  # noqa: E402  (imports the reference from a temp copy)

from compressed_tensors.quantization import QuantizationArgs, QuantizationStatus, preset_name_to_scheme  # noqa: E402
from compressed_tensors.quantization.lifecycle.forward import forward_quantize  # noqa: E402
from compressed_tensors.quantization.utils import compute_dynamic_scales_and_zp, generate_gparam  # noqa: E402

SEED = 20261016
PRESETS = ["FP8_DYNAMIC", "W8A8", "W4A8", "W4AFP8", "FP8_BLOCK", "NVFP4", "MXFP4", "MXFP8"]
CUSTOM = {
    "INT8_TOKEN_ASYM": dict(num_bits=8, type="int", strategy="token", symmetric=False, dynamic=True),
    "INT8_TENSOR_ASYM": dict(num_bits=8, type="int", strategy="tensor", symmetric=False, dynamic=True),
}
TOKEN_SHAPES = [(2, 8, 256), (2, 3, 4, 64), (16, 512), (3, 5, 1032)]
GROUP_SHAPES = [(2, 8, 256), (2, 3, 4, 128), (13, 384), (3, 7, 1152)]
WIDE = (1, 2, 32768)
WIDE_SCHEMES = ("FP8_DYNAMIC", "W8A8", "INT8_TOKEN_ASYM", "NVFP4", "MXFP4")
FP4_TIES = [6.0, 0.25, 0.75, 1.25, 1.75, 2.5, 3.5, 5.0, -0.25, -0.75, -1.25, -1.75, -2.5, -3.5, -5.0, -0.0]
FP8_TIES = [448.0, 1.0625, 1.1875, 17.0, 19.0, -1.0625, -0.0, 0.0, 0.5625, -17.0, 2.125, 36.0, -38.0, 0.0029296875, -0.0, 3.25]


def make_input(shape, dtype, gen):
    x = torch.randn(shape, generator=gen) * 2
    x = torch.where(torch.rand(shape, generator=gen) < 0.01, x * 50, x)
    x2 = x.view(-1, shape[-1])
    if x2.shape[0] >= 4:
        cols = shape[-1]
        x2[0] = 0.0
        tiny = (2.0 ** -133) if dtype == torch.bfloat16 else (2.0 ** -24)
        x2[1] = tiny * torch.randint(-8, 9, (cols,), generator=gen).float()
        x2[2] = torch.tensor(FP4_TIES * 2).repeat(cols // 32 + 1)[:cols]
        x2[3] = torch.tensor(FP8_TIES * 2).repeat(cols // 32 + 1)[:cols]
    return x.to(dtype)


def scheme_args(name):
    if name in CUSTOM:
        return QuantizationArgs(**CUSTOM[name])
    return preset_name_to_scheme(name, ["Linear"]).input_activations


def main():
    gen = torch.Generator().manual_seed(SEED)
    inputs, cases = [], []
    index = {}
    for dtype in (torch.bfloat16, torch.float16):
        for shape in sorted(set(TOKEN_SHAPES + GROUP_SHAPES + [WIDE])):
            index[(shape, dtype)] = len(inputs)
            inputs.append(make_input(shape, dtype, gen))
    for name in PRESETS + list(CUSTOM):
        args = scheme_args(name)
        grouped = args.strategy in ("group", "tensor_group")
        shapes = (GROUP_SHAPES if grouped else TOKEN_SHAPES) + ([WIDE] if name in WIDE_SCHEMES else [])
        for dtype in (torch.bfloat16, torch.float16):
            for shape in shapes:
                i = index[(shape, dtype)]
                x = inputs[i]
                gscales = [None]
                if name == "NVFP4":
                    gscales = [torch.ones(1), generate_gparam(x.float().amin(), x.float().amax())]
                for gs in gscales:
                    module = torch.nn.Module()
                    module.quantization_status = QuantizationStatus.FROZEN
                    if gs is not None:
                        module.input_global_scale = gs
                    scale, zp = compute_dynamic_scales_and_zp(value=x, args=args, module=module, global_scale=gs)
                    out = forward_quantize(module, x, "input", args)
                    cases.append(dict(scheme=name, args=dict(CUSTOM.get(name, {})), input=i, global_scale=gs, scale=scale, zero_point=zp,
                                      out=out))
    mg.save("dynamic.pt", dict(inputs=inputs, cases=cases))


if __name__ == "__main__":
    main()
