#!/usr/bin/env python
"""
Exhaustive golden vectors for the FP4 (E2M1) and MX paths, produced by importing the reference exactly like make_golden.py does.
Every bf16 and every fp16 bit pattern goes through:

  quantize (NVFP4, tensor_group 16, float32 global scale)   quantization/lifecycle/forward_helpers.py:525-547, stored as the nibbles
                                                            of pack_fp4_to_uint8 (compressors/nvfp4/helpers.py:108-158)
  quantize (MXFP4, group 32, scale in the x dtype)          same, no global scale
  compress_mx_scale                                         compressors/mx_utils.py:18-31
  calculate_qparams (NVFP4 with a global scale, and MXFP4)  quantization/utils/helpers.py:50-137: one group per non-negative max |x|
                                                            (every positive finite pattern, 0 and +inf), one-sided and two-sided

and every packed byte times every scale byte goes through NVFP4PackedCompressor.decompress (e4m3 scales, two global scales) and
MXFP4PackedCompressor.decompress (E8M0 scales); decompress_mx_scale of all 256 bytes.  Codes made from NaN inputs are stored as the
reference leaves them but are undefined there and not compared.

    python tests/golden/make_golden_fp4_sweep.py   ->  tests/golden/fp4_sweep.pt.gz (and .partN.pt.gz)
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg  # noqa: E402  (imports the reference from a temp copy)

from compressed_tensors.compressors.mx_utils import compress_mx_scale, decompress_mx_scale  # noqa: E402
from compressed_tensors.compressors.mxfp4.base import MXFP4PackedCompressor  # noqa: E402
from compressed_tensors.compressors.nvfp4.base import NVFP4PackedCompressor  # noqa: E402
from compressed_tensors.compressors.nvfp4.helpers import pack_fp4_to_uint8  # noqa: E402
from compressed_tensors.quantization import QuantizationArgs, QuantizationScheme  # noqa: E402
from compressed_tensors.quantization.lifecycle.forward import quantize  # noqa: E402
from compressed_tensors.quantization.utils import calculate_qparams  # noqa: E402

F8 = torch.float8_e4m3fn
DTS = {"bf16": torch.bfloat16, "fp16": torch.float16}
NV = dict(num_bits=4, type="float", symmetric=True, strategy="tensor_group", group_size=16, scale_dtype=F8, zp_dtype=F8)
MX4 = dict(num_bits=4, type="float", symmetric=True, strategy="group", group_size=32, scale_dtype=torch.uint8, zp_dtype=torch.uint8)
GS_384 = 2688.0 / 7.0                                  # 448 * 6 / 7: the global scale of a tensor whose max |x| is 7

# (e4m3 scale value, float32 global scale, fp8 zero point or None).  Chosen so that quotients land on every E2M1 tie and one float32
# ulp either side: a power-of-two s_eff puts x = tie * s_eff exactly on a tie, the s_eff next to 1, 7/6 and 0.875 + 2^-24 move
# quotients one float32 ulp off a tie (tests/test_fp4_sweep_host.py counts them).
NV_CASES = [
    (1.0, 1.0, None),
    (6.0, GS_384, None),                               # s_eff = 2^-6
    (448.0, GS_384, None),                             # s_eff = RN(7/6)
    (0.001953125, 1.0, None),                          # the smallest e4m3 subnormal, 2^-9
    (0.125, 2.0 ** 20, None),                          # s_eff = 2^-23
    (3.5, 1.0, None),
    (1.0, 1.0 - 2.0 ** -24, None),                     # s_eff = 1 + 2^-23 after rounding
    (1.0, 1.0 + 2.0 ** -23, None),                     # s_eff = 1 - 2^-24 after rounding
    (0.01171875, 0.011718750931322575, None),          # s_eff = 1 - 2^-24
    (0.01171875, 0.01339285634458065, None),           # s_eff = 0.875 + 2^-24
    (448.0, 2.0 ** -10, None),                         # s_eff = 448 * 2^10: everything below 2^20 rounds to zero
    (1.0, 7.0, None),                                  # s_eff = RN(1/7): quotients that only the float32 rounding of s_eff moves off a tie
    (1.5, 3.0, -0.5),                                  # s_eff = 0.5 with a zero point
    (0.75, 1.0, 4.0),
]
# (scale value, uint8 zero point or None).  Powers of two and two values that are not (the reference takes any float scale)
MX_CASES = [(2.0 ** -20, None), (2.0 ** -6, None), (0.5, None), (1.0, None), (2.0, None), (8.0, None), (128.0, None),
            (2.0 ** 14, None), (0.3, None), (1.7, None), (1.0, 1)]
QP_GS = [1.0, GS_384, 2.0 ** 40]
DQ_GS = [1.0, GS_384]


def every_pattern(dt):
    """the 65536 values of dt, bit pattern p at index p"""
    return torch.arange(65536, dtype=torch.int32).to(torch.int16).view(dt)


def positive_maxima(dt):
    """every positive finite pattern of dt in ascending order, then 0 and +inf"""
    x = every_pattern(dt)[: 1 << 15]
    return torch.cat([x[1:][x[1:].isfinite()], torch.tensor([0.0, float("inf")], dtype=dt)])


def main():
    cases = []
    nv_args, mx_args = QuantizationArgs(**NV), QuantizationArgs(**MX4)

    for name, dt in DTS.items():
        x = every_pattern(dt).reshape(1024, 64)
        for s, gs, zp in NV_CASES:
            scale = torch.full((1024, 4), s, dtype=torch.float32)
            gst = torch.tensor([gs], dtype=torch.float32)
            z = None if zp is None else torch.full((1024, 4), zp).to(F8)
            q = quantize(x, scale, z, nv_args, global_scale=gst)
            cases.append(dict(kind="nvfp4_quantize", dtype=name, scale=s, global_scale=gst, zero_point=zp, packed=pack_fp4_to_uint8(q)))

    for name, dt in DTS.items():
        x = every_pattern(dt).reshape(1024, 64)
        for s, zp in MX_CASES:
            scale = torch.full((1024, 2), s, dtype=dt)
            z = None if zp is None else torch.full((1024, 2), zp, dtype=torch.uint8)
            q = quantize(x, scale, z, mx_args)
            cases.append(dict(kind="mxfp4_quantize", dtype=name, scale=float(scale[0, 0]), zero_point=zp, packed=pack_fp4_to_uint8(q)))

    for name, dt in DTS.items():
        cases.append(dict(kind="compress_mx_scale", dtype=name, code=compress_mx_scale(every_pattern(dt), torch.uint8)))
    cases.append(dict(kind="decompress_mx_scale", value=decompress_mx_scale(torch.arange(256, dtype=torch.int32).to(torch.uint8))))

    for name, dt in DTS.items():
        m = positive_maxima(dt)
        zeros = torch.zeros_like(m)
        for sided, mn, mxv in (("one", zeros, m), ("two", -m, (m.float() * 0.5).to(dt))):
            for gs in QP_GS:
                scale, _ = calculate_qparams(mn, mxv, nv_args, global_scale=torch.tensor([gs], dtype=torch.float32))
                cases.append(dict(kind="nvfp4_qparams", dtype=name, sided=sided, global_scale=gs, scale=scale.to(F8).view(torch.uint8)))
            scale, _ = calculate_qparams(mn, mxv, mx_args)
            cases.append(dict(kind="mxfp4_qparams", dtype=name, sided=sided, global_scale=None, scale=scale))

    packed = torch.arange(256, dtype=torch.int32).to(torch.uint8).repeat(256, 1)      # row r: every byte, under scale byte r
    rows = torch.arange(256, dtype=torch.int32).to(torch.uint8)
    for gs in DQ_GS:
        scheme = QuantizationScheme(targets=["Linear"], weights=nv_args)
        state = {"weight_packed": packed, "weight_scale": rows[:, None].repeat(1, 32).view(F8), "weight_global_scale": torch.tensor([gs])}
        cases.append(dict(kind="nvfp4_decompress", global_scale=gs, weight=NVFP4PackedCompressor.decompress(state, scheme)["weight"]))
    scheme = QuantizationScheme(targets=["Linear"], weights=mx_args)
    state = {"weight_packed": packed, "weight_scale": rows[:, None].repeat(1, 16)}
    cases.append(dict(kind="mxfp4_decompress", global_scale=None, weight=MXFP4PackedCompressor.decompress(state, scheme)["weight"]))
    mg.save("fp4_sweep.pt", {"cases": cases})


if __name__ == "__main__":
    main()
