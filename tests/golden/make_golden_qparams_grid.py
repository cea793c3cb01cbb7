#!/usr/bin/env python
"""
Golden values of the memoryless min-max observer rule, calculate_qparams (quantization/utils/helpers.py:50-137), on every finite
(min, max) pair of bf16 and fp16, produced by importing the reference exactly like make_golden.py does.  The grid is
tests/qparams_model.py's: min runs over +0, -0 and every negative finite pattern, max over +0 and every positive finite pattern,
each in ascending bit-pattern order (about 1.07e9 pairs for bf16 and 1.01e9 for fp16).  Configs: int4 / int8 symmetric and
asymmetric (int8 zero points) and FP8 (e4m3) symmetric.

  sym      symmetric configs depend only on max |.|: the scale of every finite magnitude m, one-sided negative (min = -m,
           max = 0) and one-sided positive (min = 0, max = m), with the zero-point bytes
  digests  asymmetric configs: one blake2b-64 row digest (tests/qparams_model.py:row_digest) per min row of the full grid
  ladder   asymmetric configs, outright scale bits and zero points: every min x each rung of LADDER as max ("max" cases), and
           every max x each rung negated as min ("min" cases)

The rungs cross the places where the rule rounds differently: subnormal scales (and scales that underflow to 0, so eps), the fp16
subnormal edge, scales on each side of 2^-100 and 2^100 (where the fused kernels switch from reciprocal to IEEE division), ranges
whose zero point ties at .5 (14.5 / 13.5 with min -0.5 / -1.5 for int4, 254.5 / 253.5 for int8, also at slow-division scales), and
max - min overflowing to inf (65504 in fp16, the largest finite bf16).

The reference evaluates about 16 M pairs in 1.5 s on an 8-core CPU, so each asymmetric digest grid takes about 2 minutes per config
and dtype, about 8 minutes in all.

    python tests/golden/make_golden_qparams_grid.py   ->  tests/golden/qparams_grid.pt.gz (and .partN.pt.gz)
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import make_golden as mg  # noqa: E402  (imports the reference from a temp copy)

from compressed_tensors.quantization import QuantizationArgs  # noqa: E402
from compressed_tensors.quantization.utils import calculate_qparams  # noqa: E402
from tests import qparams_model as M  # noqa: E402

F8 = torch.float8_e4m3fn
LADDER = [0.0, 2.0 ** -24, 2.0 ** -20, 6.097555160522461e-05, 2.0 ** -14, 14.5 * 2.0 ** -110, 15.0 * 2.0 ** -100,
          254.5 * 2.0 ** -110, 0.5, 1.0, 13.5, 14.5, 253.5, 254.5, 15.0 * 2.0 ** 100, 14.5 * 2.0 ** 105, 65504.0, 3.3895313892515355e38]
ROWS_PER_BATCH = 512


def args_of(config):
    qmin, qmax, symmetric, _ = M.CONFIGS[config]
    if config.startswith("fp8"):
        return QuantizationArgs(num_bits=8, type="float", symmetric=True, strategy="channel")
    return QuantizationArgs(num_bits=4 if config.startswith("int4") else 8, type="int", symmetric=symmetric, strategy="channel")


def ladder_bits(dt):
    """the finite, distinct patterns of dt nearest to LADDER, ascending"""
    b = M.float_to_bits(M.rn(np.array(LADDER), dt), dt)
    b = b[np.isfinite(M.bits_to_float(b, dt))]
    return np.unique(b)


def as_dt(bits, dt):
    return torch.from_numpy(np.ascontiguousarray(bits, dtype=np.uint16).view(np.int16)).view(M.TORCH_DT[dt])


def reference(mn_bits, mx_bits, dt, config):
    """(scale bit patterns as int16, zero-point bytes as uint8) of the reference on broadcast min / max patterns"""
    scale, zp = calculate_qparams(as_dt(mn_bits, dt), as_dt(mx_bits, dt), args_of(config))
    assert scale.dtype == M.TORCH_DT[dt] and zp.dtype in (torch.int8, F8)
    return scale.view(torch.int16).clone(), zp.view(torch.uint8).clone()


def main():
    cases = []
    for dt in M.TORCH_DT:
        mags = M.maxima_bits(dt)
        zeros = np.zeros_like(mags)
        for config in M.SYM:
            for side, mn, mx in (("neg", mags | np.uint16(0x8000), zeros), ("pos", zeros, mags)):
                s, z = reference(mn, mx, dt, config)
                cases.append(dict(kind="sym", dtype=dt, config=config, side=side, scale=s, zp=z))
    for dt in M.TORCH_DT:
        mins, maxs = M.minima_bits(dt), M.maxima_bits(dt)
        rungs = ladder_bits(dt)
        for config in M.ASYM:
            for r in rungs:
                s, z = reference(mins, np.full_like(mins, r), dt, config)
                cases.append(dict(kind="ladder", dtype=dt, config=config, side="max", rung=int(r), scale=s, zp=z))
                s, z = reference(np.full_like(maxs, r | 0x8000), maxs, dt, config)
                cases.append(dict(kind="ladder", dtype=dt, config=config, side="min", rung=int(r | 0x8000), scale=s, zp=z))
            rows = []
            for i in range(0, len(mins), ROWS_PER_BATCH):
                mn = np.repeat(mins[i:i + ROWS_PER_BATCH], len(maxs))
                mx = np.tile(maxs, len(mn) // len(maxs))
                s, z = reference(mn, mx, dt, config)
                rows.append(M.digests(s.numpy().view(np.uint16).reshape(-1, len(maxs)), z.numpy().view(np.int8).reshape(-1, len(maxs))))
                print(f"{dt} {config}: {i + len(mn) // len(maxs)} / {len(mins)} rows", end="\r", flush=True)
            print()
            cases.append(dict(kind="digests", dtype=dt, config=config, digests=torch.from_numpy(np.concatenate(rows))))
    mg.save("qparams_grid.pt", {"ladder": [float(v) for v in LADDER], "cases": cases})


if __name__ == "__main__":
    main()
