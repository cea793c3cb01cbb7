#!/usr/bin/env python
"""
Golden vectors for the fused BLOCK and MX weight observers: the reference's calculate_qparams on each block's / group's min / max, then
the compressor body the preset names (NaiveQuantizationCompressor.compress for FP8_BLOCK -- its padding to whole blocks, quantize and
truncation -- and MXFP4PackedCompressor / MXFP8QuantizationCompressor.compress for the MX presets), by importing the reference exactly
like make_golden.py does.

    python tests/golden/make_golden_observe_block_mx.py   ->  tests/golden/observe_block_mx.pt.gz

Weights are bf16 and fp16 randn with 1 % outliers at 50x.  Shapes: exact and ragged ([300, 200] in 128 x 128 blocks, [257, 96] for
MX), the non-square block structures [64, 128], [128, 64], [32, 256] and [16, 40] (40 columns: no fused kernel, the unfused path), and
rows of the width of Llama-3-8B's weights (4096 and 14336).  Specials: an all-zero block / group (the eps or unit scale), a row of
subnormals (fp16 MX scales underflow and become 1), a block with an inf, and for BLOCK a block with a NaN (NaN scale; the codes made
from it are not compared).  MX cases carry no NaN: the reference's power-of-two rounding works on the NaN's bits, whichever NaN its
reduction returns.
"""
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg  # noqa: E402  (imports the reference from a temp copy)

from compressed_tensors.compressors import BaseCompressor  # noqa: E402
from compressed_tensors.quantization import QuantizationArgs, preset_name_to_scheme  # noqa: E402
from compressed_tensors.quantization.utils import calculate_qparams  # noqa: E402

SEED = 20261017
BLOCK_CASES = [((128, 256), [128, 128]), ((300, 200), [128, 128]), ((128, 128), [64, 128]), ((136, 72), [128, 64]),
               ((64, 264), [32, 256]), ((48, 120), [16, 40]), ((2, 4096), [128, 128])]
MX_SHAPES = [(32, 256), (257, 96), (3, 1024), (1, 14336)]


def make_weight(shape, dtype, gen, specials):
    x = torch.randn(shape, generator=gen) * 0.05
    x = torch.where(torch.rand(shape, generator=gen) < 0.01, x * 50, x)
    rows, cols = shape
    if specials and rows >= 8:
        x[rows - 1] = 0.0                                                    # an all-zero last row: zero blocks / groups
        tiny = (2.0 ** -133) if dtype == torch.bfloat16 else (2.0 ** -24)
        x[rows - 2] = tiny * torch.randint(-8, 9, (cols,), generator=gen).float()
        x[1, 3] = float("inf")
    return x.to(dtype)


def block_case(shape, block, dtype, gen):
    x = make_weight(shape, dtype, gen, specials=True)
    if shape[0] >= 8:
        x[shape[0] // 2, 5] = float("nan")
    scheme = preset_name_to_scheme("FP8_BLOCK", ["Linear"])
    scheme.weights = QuantizationArgs(num_bits=8, type="float", strategy="block", symmetric=True, dynamic=False, block_structure=block)
    bh, bw = block
    nrb, ncb = math.ceil(shape[0] / bh), math.ceil(shape[1] / bw)
    xp = torch.nn.functional.pad(x, (0, ncb * bw - shape[1], 0, nrb * bh - shape[0])).reshape(nrb, bh, ncb, bw)
    scale, _ = calculate_qparams(xp.amin(dim=(1, 3)), xp.amax(dim=(1, 3)), scheme.weights)
    out = BaseCompressor.load_from_registry("float-quantized").compress({"weight": x, "weight_scale": scale}, scheme)
    return {"kind": "block", "x": x, "block": list(block), "scale": scale, "weight": out["weight"]}


def mx_case(preset, shape, dtype, gen):
    x = make_weight(shape, dtype, gen, specials=True)
    scheme = preset_name_to_scheme(preset, ["Linear"])
    g = x.unflatten(-1, (-1, 32))
    scale, _ = calculate_qparams(g.amin(-1), g.amax(-1), scheme.weights)
    fmt = "mxfp4-pack-quantized" if scheme.weights.num_bits == 4 else "mxfp8-quantized"
    out = BaseCompressor.load_from_registry(fmt).compress({"weight": x, "weight_scale": scale}, scheme)
    q = out["weight_packed"] if scheme.weights.num_bits == 4 else out["weight"]
    return {"kind": "mx", "preset": preset, "num_bits": scheme.weights.num_bits, "x": x, "scale_float": scale,
            "scale": out["weight_scale"], "q": q}


def main():
    gen = torch.Generator().manual_seed(SEED)
    cases = []
    for dtype in (torch.bfloat16, torch.float16):
        for shape, block in BLOCK_CASES:
            cases.append(block_case(shape, block, dtype, gen))
        for preset in ("MXFP4", "MXFP8"):
            for shape in MX_SHAPES:
                cases.append(mx_case(preset, shape, dtype, gen))
    for c in cases:
        assert all(isinstance(v, (torch.Tensor, int, float, str, list)) for v in c.values())
    mg.save("observe_block_mx.pt", cases)


if __name__ == "__main__":
    main()
