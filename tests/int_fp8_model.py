"""
A float64 model of the reference's integer and FP8 quantize / dequantize arithmetic, written from the reference's Python and
independent of oracle/ and csrc/ (the FP4 / MX counterpart is tests/e2m1_model.py, whose roundings it reuses).  Each torch op of the
reference is one explicit rounding to the dtype it evaluates in.  A bf16 / fp16 op of ATen widens to float32, operates and narrows,
so an op in T is RN_T(RN_f32(exact)): float64 holds the exact sum, difference or product of two values of at most 24 bits, and
rounds a quotient of two such values once more without changing what RN_f32 gives (53 >= 2 * 24 + 2).  Reference paths are under
src/compressed_tensors:

  quantize        forward_helpers.py:523-547   T(fp32(x) / fp32(s)); + zp.to(T); quant_args.py:460-496 clamp(qmin, qmax) in T;
                                               torch.round (half to even, round(-0.3) = -0.0) or .to(float8_e4m3fn); .to(T)
  dequantize      forward_helpers.py:550-571   (q.to(S) - zp.to(S)) * s, both rounded to the scale dtype S
  fake_quantize   forward_helpers.py:181-215   the two above without the intermediate code dtype
  pack_to_int32   pack_quantized/helpers.py:20-101   row r's bit stream is sum_j (code_j + 2^(B-1)) << (j * B), cut into int32 words

Values are numpy float64 arrays holding values of the named dtype ("bf16", "fp16" or "f32"); e4m3 codes are uint8 bytes.
"""
import numpy as np

from tests.e2m1_model import bits_to_float, e4m3_decode, rn  # noqa: F401  (re-exported for the tests)

E4M3_MAX = 448.0


def q_range(kind, bits):
    """(qmin, qmax) of quant_args.py:calculate_range: [-2^(B-1), 2^(B-1) - 1] for integers, +-448 for float8_e4m3fn"""
    if kind == "fp8":
        return -E4M3_MAX, E4M3_MAX
    return -float(1 << (bits - 1)), float((1 << (bits - 1)) - 1)


def op(v, dt):
    """one ATen op in dt: the exact (float64) result rounded to float32, then to dt"""
    return rn(rn(v, "f32"), dt)


def quotient(x, s, dt):
    """scaled = x / scale in the x dtype dt"""
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        return op(np.asarray(x, np.float64) / np.asarray(s, np.float64), dt)


def add_zp(q, zp, dt):
    """scaled += zero_point.to(dt); int8 and e4m3 zero points are exact in every dt, -0.0 included"""
    if zp is None:
        return np.asarray(q, np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        return op(np.asarray(q, np.float64) + np.asarray(zp, np.float64), dt)


def clamp(t, lo, hi):
    """torch.clamp: NaN stays NaN, the sign of zero is kept"""
    t = np.asarray(t, np.float64)
    return np.where(np.isnan(t), t, np.minimum(np.maximum(t, lo), hi))


def e4m3_cast(v):
    """Tensor.to(float8_e4m3fn) of float values: round to nearest, ties to the even byte; 448 < |v| <= 464 gives 448 (464 is the tie
    between 448 and the NaN byte, whose mantissa is odd), anything larger, inf and NaN the NaN byte 0x7F with v's sign"""
    v = np.asarray(v, np.float64)
    grid = e4m3_decode(np.arange(127))                           # 0 .. 448 ascending
    a = np.abs(v)
    hi = np.clip(np.searchsorted(grid, np.minimum(a, E4M3_MAX)), 1, 126)
    lo = hi - 1
    dlo, dhi = a - grid[lo], grid[hi] - a
    b = np.where((dhi < dlo) | ((dhi == dlo) & (hi % 2 == 0)), hi, lo)
    b = np.where(a > E4M3_MAX, np.where(a <= 464.0, 126, 127), b)
    b = np.where(np.isnan(v), 127, b)
    return (b | (np.signbit(v).astype(np.int64) << 7)).astype(np.uint8)


def round_code(t, kind):
    """round_to_quantized_type_args after the clamp, cast back to the float dtype (every result is exact in bf16 and fp16)"""
    if kind == "fp8":
        return e4m3_decode(e4m3_cast(t))
    return np.round(t)                                           # half to even, -0.0 kept, NaN kept


def quantize(x, s, dt, kind, bits, zp=None):
    """quantized_ground of _quantize in dt, before the final .to(int8 / float8_e4m3fn)"""
    lo, hi = q_range(kind, bits)
    return round_code(clamp(add_zp(quotient(x, s, dt), zp, dt), lo, hi), kind)


def int_codes(v):
    """.to(int8) of integer-valued floats; NaN (undefined in the reference) gives 0"""
    return np.nan_to_num(np.asarray(v, np.float64), nan=0.0).astype(np.int64).astype(np.int8)


def fp8_bytes(v):
    """.to(float8_e4m3fn) of values already on the e4m3 grid (NaN stays the NaN byte)"""
    return e4m3_cast(v)


def dequantize(q, s, sdt, zp=None):
    """_dequantize: q.to(S), - zp.to(S), * scale, each in the scale dtype S.  q: code values (int8 values, or decoded e4m3 values)"""
    v = op(np.asarray(q, np.float64), sdt)
    with np.errstate(invalid="ignore", over="ignore"):
        if zp is not None:
            v = op(v - np.asarray(zp, np.float64), sdt)
        return op(v * np.asarray(s, np.float64), sdt)


def fake_quantize(x, s, dt, kind, bits, zp=None):
    """_quantize_dequantize with scale, zero point and x of dtype dt"""
    return dequantize(quantize(x, s, dt, kind, bits, zp), s, dt, zp)


def pack_int32(codes, bits):
    """pack_to_int32(packed_dim=1) of a 2-D int8 code array: element j of a row holds bits [j * B, j * B + B) of the row's stream
    (word j * B // 32, spilling into the next word), as code + 2^(B-1); rows are padded with zero bits to whole words"""
    codes = np.asarray(codes).astype(np.int64)
    rows, cols = codes.shape
    words = -(-cols * bits // 32)
    u = (codes + (1 << (bits - 1))).astype(np.uint64)
    pos = np.arange(cols, dtype=np.int64) * bits
    w, off = pos // 32, (pos % 32).astype(np.uint64)
    out = np.zeros((rows, words + 1), dtype=np.uint64)
    np.add.at(out, (slice(None), w), (u << off) & np.uint64(0xFFFFFFFF))
    spill = (pos % 32) + bits > 32
    if spill.any():
        np.add.at(out, (slice(None), w[spill] + 1), u[:, spill] >> (np.uint64(32) - off[spill]))
    return (out[:, :words] & np.uint64(0xFFFFFFFF)).astype(np.uint32).view(np.int32)
