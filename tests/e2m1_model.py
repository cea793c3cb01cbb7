"""
A float64 model of the reference's FP4 (E2M1) and MX arithmetic, written from the reference's Python and independent of oracle/ and
csrc/.  Every rounding the reference performs is made explicit: a value is computed exactly (or to float64, whose 53 bits make the
following single rounding exact for a quotient or product of two values of at most 24 bits) and then rounded once to the dtype the
reference evaluates in.  Reference paths are under src/compressed_tensors.

Inputs and outputs are numpy float64 arrays holding values of the named dtype ("bf16", "fp16" or "f32"), or uint8 / uint16 bit
patterns where a function says so.
"""
import numpy as np

LEVELS = np.array([0.0, 0.5, 1.0, 1.5, 2.0, 3.0, 4.0, 6.0])
TIES = (0.25, 0.75, 1.25, 1.75, 2.5, 3.5, 5.0)


def rn(v, dt):
    """round float64 values to the nearest `dt` value, ties to even (overflow to inf, NaN kept)"""
    v = np.asarray(v, dtype=np.float64)
    if dt == "f64":
        return v
    if dt == "fp16":
        return v.astype(np.float16).astype(np.float64)
    f = v.astype(np.float32)
    if dt == "f32":
        return f.astype(np.float64)
    assert dt == "bf16", dt
    b = f.view(np.uint32).astype(np.uint64)
    r = ((b + 0x7FFF + ((b >> 16) & 1)) >> 16) & 0xFFFF          # round to nearest even on the float32 bits (24 >= 2 * 8 + 2)
    r = np.where(np.isnan(f), (b >> 16) | 0x40, r)               # NaN stays NaN
    return bits_to_float(r.astype(np.uint16), "bf16")


def bits_to_float(bits, dt):
    """uint16 bit patterns -> float64 values of bf16 / fp16"""
    bits = np.asarray(bits, dtype=np.uint16)
    if dt == "fp16":
        return bits.view(np.float16).astype(np.float64)
    return (bits.astype(np.uint32) << 16).view(np.float32).astype(np.float64)


def e2m1(q):
    """quant_args.py:481 torch.clamp(q, -6, 6), then fp4_utils.py:88-98 cast_to_fp4: ties 0.25, 1.25, 2.5, 5.0 go down and 0.75,
    1.75, 3.5 go up; the result is |level| * torch.sign(q), so q = +-0.0 gives +0.0, a negative q that rounds to zero -0.0, NaN NaN"""
    q = np.clip(q, -6.0, 6.0)
    a = np.abs(q)
    v = np.select([a <= 0.25, a < 0.75, a <= 1.25, a < 1.75, a <= 2.5, a < 3.5, a <= 5.0], LEVELS[:7].tolist(), 6.0)
    sign = np.where(q > 0, 1.0, np.where(q < 0, -1.0, 0.0))
    return np.where(np.isnan(q), np.nan, np.where(sign == 0, 0.0, v * sign))


def nvfp4_quotient(x, scale, gs, zp=None):
    """forward_helpers.py:535-540 with a float32 global scale: s_eff = RN_f32(scale / gs); q = RN_f32(x / s_eff) (x / scale promotes
    to float32); q += zp.to(x.dtype) in float32"""
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        s_eff = rn(np.asarray(scale, np.float64) / np.float64(gs), "f32")
        q = rn(np.asarray(x, np.float64) / s_eff, "f32")
        return q if zp is None else rn(q + zp, "f32")


def nvfp4_quantize(x, scale, gs, zp=None):
    """forward_helpers.py:525-547: the quotient above through the E2M1 ladder"""
    return e2m1(nvfp4_quotient(x, scale, gs, zp))


def mx_quotient(x, scale, dt, zp=None):
    """forward_helpers.py:538-540 without a global scale, x and scale both of dtype dt: q = RN_dt(x / scale); q += zp.to(dt) in dt"""
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        q = rn(np.asarray(x, np.float64) / np.asarray(scale, np.float64), dt)
        return q if zp is None else rn(q + zp, dt)


def mx_quantize(x, scale, dt, zp=None):
    """the quotient above through the E2M1 ladder (every threshold and level is a dt value, so the ladder needs no rounding)"""
    return e2m1(mx_quotient(x, scale, dt, zp))


def fp4_value(code):
    """compressors/nvfp4/helpers.py:162-193: nibble -> value; bit 3 is the sign (code 8 is -0.0)"""
    code = np.asarray(code).astype(np.int64)
    v = LEVELS[code & 7]
    return np.where(code & 8, -v, v)


def unpack_nibbles(packed):
    """helpers.py:185-188: byte i of a row holds element 2i in its low nibble and element 2i + 1 in its high nibble"""
    packed = np.asarray(packed, dtype=np.uint8)
    out = np.empty(packed.shape[:-1] + (packed.shape[-1] * 2,), dtype=np.uint8)
    out[..., 0::2] = packed & 0xF
    out[..., 1::2] = packed >> 4
    return out


def pack_nibbles(v):
    """helpers.py:108-158 on valid E2M1 values (-0.0 keeps its sign bit): low nibble = even element, high nibble = odd element"""
    v = np.asarray(v, dtype=np.float64)
    idx = np.searchsorted(LEVELS, np.abs(v)).astype(np.uint8) | (np.signbit(v).astype(np.uint8) << 3)
    return (idx[..., 0::2] | (idx[..., 1::2] << 4)).astype(np.uint8)


def fp4_dequantize(code, scale, gs, out_dt):
    """forward_helpers.py:550-571 on unpacked E2M1 values held in scale's dtype T.  With a float32 global scale:
    RN_T(RN_f32(RN_f32(scale / gs) * v)); without one: RN_T(v * scale)"""
    v = fp4_value(code)
    with np.errstate(invalid="ignore", over="ignore"):
        if gs is None:
            return rn(v * np.asarray(scale, np.float64), out_dt)
        s_eff = rn(np.asarray(scale, np.float64) / np.float64(gs), "f32")
        return rn(rn(s_eff * v, "f32"), out_dt)


def round_to_power_2(bits, dt):
    """mxfp_utils.py:70-120 on uint16 patterns: (x + (1 << (mantissa - 2))) & sign-and-exponent mask, in int32, truncated to 16 bits"""
    mant, expo = (7, 8) if dt == "bf16" else (10, 5)
    x = np.asarray(bits, dtype=np.uint16).astype(np.int64)
    mask = ((1 << (expo + 1)) - 1) << mant
    return ((x + (1 << (mant - 2))) & mask).astype(np.uint16)


def e4m3_decode(byte):
    """float8_e4m3fn: bias 7, subnormals 2^-6 * m / 8, 0x7F / 0xFF NaN, no infinities"""
    b = np.asarray(byte, dtype=np.int64)
    e, m = (b >> 3) & 0xF, b & 7
    mag = np.where(e == 0, np.ldexp(m / 8.0, -6), np.ldexp(1.0 + m / 8.0, e - 7))
    mag = np.where((b & 0x7F) == 0x7F, np.nan, mag)
    return np.where(b & 0x80, -mag, mag)


def e4m3_encode(v):
    """float32 values within [-448, 448] -> the nearest float8_e4m3fn byte, ties to the even byte (torch's .to(float8_e4m3fn))"""
    v = np.asarray(v, dtype=np.float64)
    grid = e4m3_decode(np.arange(127))                          # 0 .. 448 ascending
    a = np.abs(v)
    hi = np.clip(np.searchsorted(grid, a), 1, 126)
    lo = hi - 1
    dlo, dhi = a - grid[lo], grid[hi] - a
    b = np.where((dhi < dlo) | ((dhi == dlo) & (hi % 2 == 0)), hi, lo)
    return (b | (np.signbit(v).astype(np.int64) << 7)).astype(np.uint8)


def nvfp4_scale_code(amax, gs, dt):
    """quantization/utils/helpers.py:79-125 for NVFP4 (symmetric, scale_dtype float8_e4m3fn) on a group's max |x| of dtype dt:
    RN_dt(amax / 6), RN_f32(gs * that), clamp to +-448, RN_e4m3; a zero scale becomes 0.125.  Returns the e4m3 byte"""
    with np.errstate(over="ignore", invalid="ignore"):
        s = rn(rn(rn(np.asarray(amax, np.float64) / 6.0, "f32"), dt) * np.float64(gs), "f32")
    code = e4m3_encode(np.clip(s, -448.0, 448.0))
    return np.where((code & 0x7F) == 0, e4m3_encode(0.125), code).astype(np.uint8)


def mx_scale(amax_bits, dt, num_bits=4):
    """quantization/utils/helpers.py:79-125 for MX (scale_dtype uint8) and mxfp_utils.py:123-142 on max |x| bit patterns of dtype dt:
    e = 127 + log2(round_to_power_2(amax)) - (2 for FP4, 8 for FP8), clamped to [0, 255]; scale = RN_dt(2^(e - 127)); zero -> 1"""
    p2 = bits_to_float(round_to_power_2(amax_bits, dt), dt)      # 0, a power of two or inf
    with np.errstate(divide="ignore"):
        e = np.clip(127 + np.log2(p2) - (2 if num_bits == 4 else 8), 0, 255)
    s = rn(rn(np.ldexp(1.0, e.astype(np.int64) - 127), "f32"), dt)
    return np.where(s == 0, 1.0, s)


def e8m0_decode(byte):
    """compressors/mx_utils.py:43-44: 2.0 ** (e - 127).to(bfloat16) -> bfloat16; 255 gives 2^128 = inf"""
    return rn(np.ldexp(1.0, np.asarray(byte, dtype=np.int64) - 127), "bf16")
