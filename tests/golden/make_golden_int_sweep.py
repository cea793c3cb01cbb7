#!/usr/bin/env python
"""
Exhaustive golden vectors for the integer and FP8 paths, produced by importing the reference exactly like make_golden.py does.
Every bf16 and every fp16 bit pattern, under each scale of SCALES (TENSOR strategy, scale and x of one dtype), goes through

  quantize        forward.py:36-73 with dtype=int8 / float8_e4m3fn (stored as int8 codes / e4m3 bytes)
  fake_quantize   forward.py:148-181 (stored as the 16-bit patterns of its output)

for each of CONFIGS: int4, int8 and int3 symmetric and asymmetric, int6 symmetric, and FP8 without a zero
point and with an fp8 zero point of +0.0 and of -0.0.  And every int8 code under every int8 zero point, and every e4m3 byte under
every e4m3 zero point byte, goes through dequantize (forward.py:76-145, CHANNEL scale: row r holds every code under zero point r) at
each scale of SCALES and in bf16, fp16 and float32.  Codes made from NaN inputs are stored as the reference leaves them but are
undefined there and not compared.  The golden also holds CONFIGS and SCALES.

    python tests/golden/make_golden_int_sweep.py   ->  tests/golden/int_sweep.pt.gz (and .partN.pt.gz)
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg  # noqa: E402  (imports the reference from a temp copy)

from compressed_tensors.quantization import QuantizationArgs  # noqa: E402
from compressed_tensors.quantization.lifecycle.forward import dequantize, fake_quantize, quantize  # noqa: E402

F8 = torch.float8_e4m3fn
DTS = {"bf16": torch.bfloat16, "fp16": torch.float16, "f32": torch.float32}

# (name, kind, bits, zero point or None).  The zero point is an int8 value, or an e4m3 value (what the FP8 presets register)
CONFIGS = [
    ("int4", "int", 4, None), ("int4_zp", "int", 4, -3), ("int8", "int", 8, None), ("int8_zp", "int", 8, 37),
    ("int3", "int", 3, None), ("int3_zp", "int", 3, 1), ("int6", "int", 6, None), ("fp8", "fp8", 8, None), ("fp8_zp+0", "fp8", 8, 0.0), ("fp8_zp-0", "fp8", 8, -0.0),
]
# Powers of two put quotients exactly on every .5 tie and e4m3 midpoint; the others move them off.  bf16 also has the neighbours of
# 2^-100 and 2^100, where the kernels switch between a reciprocal and IEEE division, and a subnormal; fp16 its extremes.
SCALES = {
    "bf16": [1.0, 2.0 ** -7, 0.01, 37.5, 0.3, -0.7, 2.0 ** -100 * (1 - 2.0 ** -8), 2.0 ** -100 * (1 + 2.0 ** -7),
             2.0 ** 100 * (1 - 2.0 ** -8), 2.0 ** 100 * (1 + 2.0 ** -7), 2.0 ** -130, 3.0e38],
    "fp16": [1.0, 2.0 ** -7, 0.01, 37.5, 0.3, -0.7, 2.0 ** -24, 2.0 ** -14, 1.7, 1000.0, 65504.0, 3.0 / 1024],
    "f32": [1.0, 0.01, 37.5, -0.7, 2.0 ** -100 * (1 - 2.0 ** -24), 2.0 ** 100 * (1 + 2.0 ** -23), 2.0 ** -140, 0.3],
}


def every_pattern(dt):
    """the 65536 values of dt, bit pattern p at index p"""
    return torch.arange(65536, dtype=torch.int32).to(torch.int16).view(dt)


def args_of(kind, bits, zp):
    if kind == "fp8":
        return QuantizationArgs(num_bits=8, type="float", symmetric=zp is None, strategy="tensor")
    return QuantizationArgs(num_bits=bits, type="int", symmetric=zp is None, strategy="tensor")


def zp_tensor(kind, zp):
    if zp is None:
        return None
    return torch.tensor([zp]).to(F8) if kind == "fp8" else torch.tensor([zp], dtype=torch.int8)


def main():
    cases = []
    for name in ("bf16", "fp16"):
        dt = DTS[name]
        x = every_pattern(dt).reshape(256, 256)
        for s in SCALES[name]:
            st = torch.tensor([s], dtype=torch.float64).to(dt)
            for cfg, kind, bits, zp in CONFIGS:
                a, z = args_of(kind, bits, zp), zp_tensor(kind, zp)
                q = quantize(x, st, z, a, dtype=F8 if kind == "fp8" else torch.int8)
                fq = fake_quantize(x, st, z, a)
                cases.append(dict(kind="quantize", dtype=name, scale=float(st), config=cfg,
                                  code=q.view(torch.uint8) if kind == "fp8" else q, fake=fq.view(torch.int16)))

    rows = torch.arange(256, dtype=torch.int32)
    int_codes = (rows - 128).to(torch.int8)[None, :].repeat(256, 1)          # row r: every int8 code, under zero point r - 128
    int_zp = (rows - 128).to(torch.int8)[:, None]
    f8_codes = rows.to(torch.uint8)[None, :].repeat(256, 1).view(F8)          # row r: every e4m3 byte, under zero point byte r
    f8_zp = rows.to(torch.uint8)[:, None].view(F8)
    for name, dt in DTS.items():
        for s in SCALES[name]:
            st = torch.full((256, 1), s, dtype=torch.float64).to(dt)
            cases.append(dict(kind="dequantize", dtype=name, scale=float(st[0, 0]), config="int8_zp",
                              value=dequantize(int_codes, st, int_zp).view(torch.int32 if name == "f32" else torch.int16)))
            cases.append(dict(kind="dequantize", dtype=name, scale=float(st[0, 0]), config="fp8_zp",
                              value=dequantize(f8_codes, st, f8_zp).view(torch.int32 if name == "f32" else torch.int16)))
    # the tables travel with the golden, so that the tests read them without importing the reference
    mg.save("int_sweep.pt", {"configs": [list(c) for c in CONFIGS], "scales": SCALES, "cases": cases})


if __name__ == "__main__":
    main()
