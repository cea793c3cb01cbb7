"""
A float64 model of the reference's memoryless min-max observer rule for integer and FP8 schemes, calculate_qparams
(quantization/utils/helpers.py:50-137), written from the reference's Python and independent of oracle/ and csrc/.  Each torch op of
the rule runs on a tensor of the min / max dtype T (bf16 or fp16), which ATen evaluates in float32 and rounds to T; the model
computes each op in float64 and rounds once to float32, then to T.  For a single +, -, * or / of values of at most 24 bits the
float64 result rounds to the same float32 as the exact one, so the double rounding is harmless.  Reference paths are under
src/compressed_tensors.

The same code runs on numpy float64 arrays (host) and on float64 torch tensors (any device): the GPU sweep evaluates it over every
(min, max) pair of a dtype.  Values are float64 holding values of T; zero points come back as int8.

The row digest defined here is what tests/golden/qparams_grid*.pt.gz stores for the full asymmetric grid, and what the host and
GPU sweeps recompute: blake2b with an 8-byte digest of one min row's scale bit patterns (uint16 little-endian) over every max in
ascending bit-pattern order, followed by the row's int8 zero-point bytes in the same order.
"""
import hashlib

import numpy as np
import torch

# name -> (qmin, qmax, symmetric, zero-point kind): quantization/utils/helpers.py:198-226 calculate_range.  FP8 is e4m3 with a
# float8 zero point, which the rule always leaves at +0.0.
CONFIGS = {
    "int4_sym": (-8.0, 7.0, True, "int8"),
    "int4_asym": (-8.0, 7.0, False, "int8"),
    "int8_sym": (-128.0, 127.0, True, "int8"),
    "int8_asym": (-128.0, 127.0, False, "int8"),
    "fp8_sym": (-448.0, 448.0, True, "fp8"),
}
ASYM = ("int4_asym", "int8_asym")
SYM = ("int4_sym", "int8_sym", "fp8_sym")
# torch.finfo(T).eps, the scale a zero one becomes (helpers.py:113-126)
EPS = {"bf16": 2.0 ** -7, "fp16": 2.0 ** -10, "f32": 2.0 ** -23}
TORCH_DT = {"bf16": torch.bfloat16, "fp16": torch.float16}

# Mutated rules, each one step wrong, so that the tests can show the golden tells every step apart (tests/test_qparams_grid_host.py)
MUTANTS = (
    "zero point rounded half away from zero",
    "max - min not rounded to T",
    "min / scale not rounded to T",
    "eps applied before the zero point",
    "* (2 / range) in place of / (range / 2)",
    "zero point not clamped to [qmin, qmax]",
)


def _torch(v):
    return isinstance(v, torch.Tensor)


def rn(v, dt):
    """round float64 values to float32 and then to dt ("f32", "bf16" or "fp16"), each time to nearest even; overflow gives inf"""
    if _torch(v):
        f = v.to(torch.float32)
        return (f if dt == "f32" else f.to(TORCH_DT[dt])).to(torch.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        f = np.asarray(v, dtype=np.float64).astype(np.float32)
        if dt == "f32":
            return f.astype(np.float64)
        if dt == "fp16":
            return f.astype(np.float16).astype(np.float64)
    assert dt == "bf16", dt
    b = f.view(np.uint32).astype(np.uint64)
    r = ((b + 0x7FFF + ((b >> 16) & 1)) >> 16) & 0xFFFF            # nearest even on the float32 bits; inf stays inf
    r = np.where(np.isnan(f), (b >> 16) | 0x40, r)
    return bits_to_float(r.astype(np.uint16), "bf16")


def bits_to_float(bits, dt):
    """uint16 bit patterns (numpy) -> float64 values of bf16 / fp16"""
    bits = np.asarray(bits, dtype=np.uint16)
    if dt == "fp16":
        return bits.view(np.float16).astype(np.float64)
    return (bits.astype(np.uint32) << 16).view(np.float32).astype(np.float64)


def float_to_bits(v, dt):
    """float64 values of bf16 / fp16 (numpy or torch) -> their uint16 bit patterns as a numpy array"""
    if _torch(v):
        return v.to(TORCH_DT[dt]).view(torch.int16).cpu().numpy().view(np.uint16)
    v = np.asarray(v, dtype=np.float64)
    with np.errstate(over="ignore"):
        if dt == "fp16":
            return v.astype(np.float16).view(np.uint16)
        return (v.astype(np.float32).view(np.uint32) >> 16).astype(np.uint16)


def maxima_bits(dt):
    """the max side of the grid: +0 and every positive finite pattern of dt, ascending"""
    top = 0x7F7F if dt == "bf16" else 0x7BFF
    return np.arange(top + 1, dtype=np.uint32).astype(np.uint16)


def minima_bits(dt):
    """the min side of the grid: +0, -0 and every negative finite pattern of dt, in ascending bit-pattern order"""
    return np.concatenate([np.zeros(1, np.uint16), maxima_bits(dt) | np.uint16(0x8000)])


def _where(c, a, b):
    return torch.where(c, a, b) if _torch(c) else np.where(c, a, b)


def _like(v, x):
    return torch.full_like(v, x) if _torch(v) else np.full_like(v, x)


def qparams(mn, mx, config, dt, mutant=None, trace=None):
    """calculate_qparams of float64 min / max values of dt for one of CONFIGS: returns (scale in dt as float64, zero point as int8;
    float8 +0.0 zero points come back as int8 0).  `mutant` picks one of MUTANTS.  `trace`, a dict, receives the intermediate values
    the coverage tests count: the rounded max - min, the scale before the eps fallback, and the zero point before and after the
    clamp to [qmin, qmax]."""
    assert mutant is None or mutant in MUTANTS, mutant
    qmin, qmax, symmetric, _ = CONFIGS[config]
    T = torch if _torch(mn) else np
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        lo = T.minimum(mn, _like(mn, 0.0))                             # :74-75, min(min, 0) and max(max, 0)
        hi = T.maximum(mx, _like(mx, 0.0))
        rng = qmax - qmin                                              # 0-dim float32 tensors: exact
        if symmetric:
            a = T.maximum(T.abs(lo), T.abs(hi))                        # :84
            if mutant == MUTANTS[4]:
                s = rn(rn(a * float(np.float32(2.0 / rng)), "f32"), dt)
            else:
                s = rn(rn(a / (rng / 2), "f32"), dt)                   # :90, the halved range is exact
            z = _like(s, 0.0)
        else:
            d = rn(rn(hi - lo, "f32"), "f32" if mutant == MUTANTS[1] else dt)     # :100
            s = rn(rn(d / rng, "f32"), dt)
            if mutant == MUTANTS[3]:
                s = _where(s == 0, _like(s, EPS[dt]), s)
            q = rn(rn(lo / s, "f32"), "f32" if mutant == MUTANTS[2] else dt)       # :101
            zu = rn(rn(qmin - q, "f32"), dt)
            z = zu if mutant == MUTANTS[5] else T.clip(zu, qmin, qmax)            # :102; NaN (0 / 0) stays NaN
            if trace is not None:
                trace.update(diff=d, raw_scale=s, z_unclamped=zu, z=z)
        s = _where(s == 0, _like(s, EPS[dt]), s)                       # :113-126
        # :129-131 round_to_quantized_type_dtype(int8): clamp to [-128, 127], round half to even, .to(int8); NaN converts to 0
        zc = T.clip(z, -128.0, 127.0)
        if mutant == MUTANTS[0]:
            r = T.sign(zc) * T.floor(T.abs(zc) + 0.5)
        else:
            r = T.round(zc)
        r = _where(r != r, _like(r, 0.0), r)
        zp = r.to(torch.int8) if _torch(r) else r.astype(np.int8)
    return s, zp


def row_digest(scale_bits, zp):
    """the digest of one min row: scale bit patterns (uint16) and int8 zero points over every max, in grid order"""
    h = hashlib.blake2b(digest_size=8)
    h.update(np.ascontiguousarray(scale_bits, dtype="<u2").tobytes())
    h.update(np.ascontiguousarray(zp, dtype=np.int8).tobytes())
    return h.digest()


def digests(scale_bits, zp):
    """row digests of a [rows, maxima] block as a uint8 array [rows, 8]"""
    return np.frombuffer(b"".join(row_digest(a, b) for a, b in zip(scale_bits, zp)), dtype=np.uint8).reshape(-1, 8)
