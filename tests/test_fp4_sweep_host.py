"""
The float64 model of tests/e2m1_model.py against the reference's own outputs on every bf16 / fp16 bit pattern
(tests/golden/fp4_sweep.pt.gz) and against the CPU oracle on the scale ladders the GPU sweep uses, so that the GPU sweep
(tests/test_gpu_fp4_sweep.py) can trust both where the golden stores nothing.

The sweep is only worth something if its inputs reach the places a rounding can go wrong, and if the comparison would see a wrong
rounding there.  So the tests also count, per dtype and per encode family, the quotients that land exactly on each of the seven
E2M1 ties and one ulp either side of each (every count must be positive), and check that the golden tells each of these mutated
models apart from the right one: 2.5 or 5.0 rounding up, 0.75 rounding down, -0.0 kept for x = -0.0, s_eff = scale / gs not
rounded to float32, scale * (1 / gs) in place of scale / gs, the nibbles swapped, an E8M0 decode one exponent off.

Dropping the clamp to +-6 before the ladder is not among them: the ladder's last rung sends everything above 5.0, infinities
included, to 6.0 with the quotient's sign, and NaN passes both, so no input tells the two apart.
"""
import numpy as np
import pytest
import torch

import oracle
from tests import e2m1_model as M
from tests.golden import load

CASES = load("fp4_sweep")["cases"]
PATTERNS = np.arange(65536, dtype=np.uint32).astype(np.uint16)
TORCH_DT = {"bf16": torch.bfloat16, "fp16": torch.float16}
GS_384 = 2688.0 / 7.0


def of(kind):
    return [c for c in CASES if c["kind"] == kind]


def case_id(c):
    return "-".join(str(c[k]) for k in ("dtype", "scale", "zero_point") if k in c) + (f"-gs{float(c['global_scale']):g}" if c.get("global_scale") is not None else "")


def every(dt):
    with np.errstate(invalid="ignore"):
        return M.bits_to_float(PATTERNS, dt)


def quotients(c):
    """the model's quotient of every pattern for golden quantize case c (before the ladder)"""
    x = every(c["dtype"])
    if c["kind"] == "nvfp4_quantize":
        return M.nvfp4_quotient(x, c["scale"], float(c["global_scale"]), c["zero_point"])
    return M.mx_quotient(x, M.rn(c["scale"], c["dtype"]), c["dtype"], c["zero_point"])


def packed_mismatches(values, c):
    """bytes of the golden's packed codes that differ from `values` packed; bytes holding a NaN input are not compared"""
    got = M.pack_nibbles(np.nan_to_num(values, nan=0.0).reshape(1024, 64))
    nan_byte = np.isnan(every(c["dtype"])).reshape(1024, 32, 2).any(-1)
    return int(((got != c["packed"].numpy()) & ~nan_byte).sum())


def mismatches(got, want):
    """bitwise float mismatches (sign of zero included), NaN matching NaN"""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    both_nan = np.isnan(got) & np.isnan(want)
    return int((((got != want) | (np.signbit(got) != np.signbit(want))) & ~both_nan).sum())


def positive_maxima_bits(dt):
    top = 0x7F80 if dt == "bf16" else 0x7C00                      # +inf
    return np.concatenate([np.arange(1, top), [0, top]]).astype(np.uint16)


# ---------------------------------------------------------------------------------------------------------------------------------
# the model against the reference's outputs
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", of("nvfp4_quantize") + of("mxfp4_quantize"), ids=lambda c: c["kind"][:5] + "-" + case_id(c))
def test_model_quantize_matches_the_golden(c):
    assert packed_mismatches(M.e2m1(quotients(c)), c) == 0
    print(f"{c['kind']} {case_id(c)}: 65536 elements")


@pytest.mark.parametrize("c", of("nvfp4_qparams") + of("mxfp4_qparams"), ids=lambda c: f"{c['kind']}-{c['dtype']}-{c['sided']}-{c['global_scale']}")
def test_model_qparams_match_the_golden(c):
    bits = positive_maxima_bits(c["dtype"])
    if c["kind"] == "nvfp4_qparams":
        assert mismatches(M.nvfp4_scale_code(M.bits_to_float(bits, c["dtype"]), c["global_scale"], c["dtype"]), c["scale"].numpy()) == 0
    else:
        assert mismatches(M.mx_scale(bits, c["dtype"]), c["scale"].float().numpy()) == 0
    print(f"{c['kind']}: {bits.size} groups")


def decompress_inputs():
    """the golden's decompress layout: row r holds every packed byte under scale byte r"""
    return M.unpack_nibbles(np.tile(np.arange(256, dtype=np.uint8), (256, 1))), np.arange(256)[:, None]


@pytest.mark.parametrize("c", of("nvfp4_decompress") + of("mxfp4_decompress"), ids=lambda c: f"{c['kind']}-{c['global_scale']}")
def test_model_decompress_matches_the_golden(c):
    code, rows = decompress_inputs()
    if c["kind"] == "nvfp4_decompress":
        got = M.fp4_dequantize(code, M.e4m3_decode(rows), c["global_scale"], "bf16")
    else:
        got = M.fp4_dequantize(code, M.e8m0_decode(rows), None, "bf16")
    assert mismatches(got, c["weight"].float().numpy()) == 0


def test_model_e8m0_decode_matches_the_golden():
    (c,) = of("decompress_mx_scale")
    assert mismatches(M.e8m0_decode(np.arange(256)), c["value"].float().numpy()) == 0


@pytest.mark.parametrize("c", of("compress_mx_scale"), ids=lambda c: c["dtype"])
def test_compress_mx_scale_golden(c):
    """the E8M0 encode takes a transcendental log2, so it is pinned by the golden rather than modelled: the oracle must reproduce it on
    every pattern, and on every positive power of two it is exactly 127 + the exponent (mod 256)"""
    dt = c["dtype"]
    code = c["code"].numpy()
    np.testing.assert_array_equal(oracle.compress_mx_scale(torch.from_numpy(PATTERNS.astype(np.int16)).view(TORCH_DT[dt])).numpy(), code)
    v = every(dt)
    pos = (v > 0) & np.isfinite(v)
    m, e = np.frexp(v[pos])
    p2 = m == 0.5
    assert p2.sum() > 0
    np.testing.assert_array_equal(code[pos][p2], ((127 + e[p2] - 1) % 256).astype(np.uint8))


# ---------------------------------------------------------------------------------------------------------------------------------
# the model against the oracle on the ladders the GPU sweep uses
# ---------------------------------------------------------------------------------------------------------------------------------
def finite_e4m3_bytes():
    b = np.arange(256)
    return b[(b & 0x7F) != 0x7F]


def oracle_values_match(x_t, s_t, want_model, **kw):
    got = oracle.quantize(x_t, s_t, None, num_bits=4, qtype="float", **kw)
    return mismatches(got.float().numpy().reshape(-1), want_model.reshape(-1))


def f32_neighbours(g):
    return [g, float(np.nextafter(np.float32(g), np.float32(0))), float(np.nextafter(np.float32(g), np.float32(np.inf)))]


# the global scales of tests/test_gpu_fp4_sweep.py's NVFP4 encode sweeps: 1 and 2688/7 for every scale byte; 2^-10 and 2^100 and their
# float32 neighbours, which put |1.0 / gs| on and either side of the ends of the fast division range [2^-100, 2^10]
@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("gs", [1.0, GS_384] + f32_neighbours(2.0 ** -10) + f32_neighbours(2.0 ** 100), ids=lambda g: f"{g:.9g}")
def test_model_matches_the_oracle_on_every_e4m3_scale(dt, gs):
    """NVFP4: every pattern at every finite e4m3 scale byte of both signs (the scale held in float32), against orc_quantize_gs; every
    eighth byte at the range-boundary global scales"""
    x = every(dt)
    xs = torch.from_numpy(PATTERNS.astype(np.int16)).view(TORCH_DT[dt]).reshape(1024, 64)
    bad = 0
    for b in finite_e4m3_bytes()[:: (1 if gs in (1.0, GS_384) else 8)]:
        s = float(M.e4m3_decode(b))
        want = M.nvfp4_quantize(x, s, gs)
        bad += oracle_values_match(xs, torch.full((1024, 4), s), want, strategy="tensor_group", group_size=16,
                                   global_scale=torch.tensor([gs], dtype=torch.float32))
    assert bad == 0


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("gs", [GS_384, 2.0 ** -10], ids=["gs384", "gs2^-10"])
@pytest.mark.parametrize("zp", [0.0, -0.0, 0.5, -1.5, 4.0, -4.0], ids=lambda z: f"{z:+g}" if z else ("-0" if np.signbit(z) else "+0"))
def test_model_matches_the_oracle_with_fp8_zero_points(dt, gs, zp):
    """NVFP4 with an fp8 zero point (-0.0 included: x = +-0.0 must still give +0.0), every eighth scale byte, the zero-point sweep's
    global scales"""
    x = every(dt)
    xs = torch.from_numpy(PATTERNS.astype(np.int16)).view(TORCH_DT[dt]).reshape(1024, 64)
    z = torch.full((1024, 4), zp).to(torch.float8_e4m3fn)
    bad = 0
    for b in finite_e4m3_bytes()[::8]:
        s = float(M.e4m3_decode(b))
        got = oracle.quantize(xs, torch.full((1024, 4), s), z, num_bits=4, qtype="float", strategy="tensor_group", group_size=16,
                              global_scale=torch.tensor([gs], dtype=torch.float32))
        bad += mismatches(got.float().numpy().reshape(-1), M.nvfp4_quantize(x, s, gs, zp))
    assert bad == 0


def mx_scale_ladder(dt):
    """every power of two dt holds, and a few values that are not"""
    lo, hi = (-133, 127) if dt == "bf16" else (-24, 15)
    return [2.0 ** e for e in range(lo, hi + 1)] + [float(M.rn(v, dt)) for v in (0.3, 1.7, 3.0, 0.011, 100.0)]


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("zp", [None, 1, 200, -3])
def test_model_matches_the_oracle_on_every_mx_scale(dt, zp):
    """MXFP4: every pattern at every power of two of the dtype and at some other scales, x dtype arithmetic, against orc_quantize_gs"""
    x = every(dt)
    xs = torch.from_numpy(PATTERNS.astype(np.int16)).view(TORCH_DT[dt]).reshape(1024, 64)
    z = None if zp is None else torch.full((1024, 2), zp, dtype=torch.uint8 if zp >= 0 else torch.int8)
    bad = 0
    for s in mx_scale_ladder(dt):
        want = M.mx_quantize(x, s, dt, zp)
        got = oracle.quantize(xs, torch.full((1024, 2), s, dtype=TORCH_DT[dt]), z, strategy="group", group_size=32, num_bits=4, qtype="float")
        bad += mismatches(got.float().numpy().reshape(-1), want)
    assert bad == 0


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_model_dequantize_matches_the_oracle(dt):
    """every code under every finite e4m3 scale with and without a global scale, and under every finite dt scale"""
    code = np.tile(np.arange(16, dtype=np.uint8), 256)
    codes_t = torch.from_numpy(M.fp4_value(code)).to(TORCH_DT[dt]).reshape(256, 16)
    s8 = M.e4m3_decode(np.arange(256))
    for gs in (None, GS_384, 2.0 ** 60, 2.0 ** -61):
        st = torch.from_numpy(s8).to(TORCH_DT[dt]).reshape(256, 1)
        want = M.fp4_dequantize(code.reshape(256, 16), M.rn(s8, dt).reshape(256, 1), gs, dt)
        got = oracle.dequantize(codes_t, st, None, strategy="group", group_size=16, dtype=TORCH_DT[dt],
                                global_scale=None if gs is None else torch.tensor([gs], dtype=torch.float32))
        assert mismatches(got.float().numpy(), want) == 0, gs
    s = every(dt)
    fin = np.isfinite(s)
    codes = np.tile(np.arange(16, dtype=np.uint8), (int(fin.sum()), 1))
    st = torch.from_numpy(PATTERNS.astype(np.int16)).view(TORCH_DT[dt])[torch.from_numpy(fin)].reshape(-1, 1)
    got = oracle.dequantize(torch.from_numpy(M.fp4_value(codes)).to(TORCH_DT[dt]), st, None, strategy="group", group_size=16, dtype=TORCH_DT[dt])
    assert mismatches(got.float().numpy(), M.fp4_dequantize(codes, s[fin][:, None], None, dt)) == 0


# ---------------------------------------------------------------------------------------------------------------------------------
# coverage and sensitivity
# ---------------------------------------------------------------------------------------------------------------------------------
def neighbours(t, dt):
    """(t one ulp below, t one ulp above) in the dtype the quotient is rounded to"""
    if dt == "f32":
        f = np.float32(t)
        return float(np.nextafter(f, np.float32(0))), float(np.nextafter(f, np.float32(np.inf)))
    if dt == "fp16":
        f = np.float16(t)
        return float(np.nextafter(f, np.float16(0))), float(np.nextafter(f, np.float16(np.inf)))
    b = int(np.float32(t).view(np.uint32)) >> 16
    return float(M.bits_to_float(b - 1, "bf16")), float(M.bits_to_float(b + 1, "bf16"))


@pytest.mark.parametrize("family", ["nvfp4_quantize", "mxfp4_quantize"])
@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_the_golden_reaches_every_tie_and_its_neighbours(family, dt):
    qdt = "f32" if family == "nvfp4_quantize" else dt
    q = np.concatenate([quotients(c) for c in of(family) if c["dtype"] == dt])
    counts = {}
    for t in M.TIES:
        below, above = neighbours(t, qdt)
        for sign in (1, -1):
            for name, v in (("below", below), ("on", t), ("above", above)):
                counts[(sign * t, name)] = int((q == sign * v).sum())
    print(f"{family} {dt}: {q.size} elements; " + ", ".join(f"{k[0]:+g} {k[1]}: {n}" for k, n in counts.items()))
    assert min(counts.values()) > 0, {k: n for k, n in counts.items() if n == 0}


def ladder(q, down=(0.25, 1.25, 2.5, 5.0), keep_negative_zero=False):
    """the E2M1 ladder with the ties in `down` rounding down and the others up"""
    q = np.clip(q, -6.0, 6.0)
    a = np.abs(q)
    v = np.full(a.shape, 6.0)
    for lo, hi, t in reversed(list(zip(M.LEVELS[:-1], M.LEVELS[1:], M.TIES))):
        v = np.where((a <= t) if t in down else (a < t), lo, v)
    v = np.where(np.signbit(q), -v, v)
    if not keep_negative_zero:
        v = np.where(q == 0, 0.0, v)
    return np.where(np.isnan(q), np.nan, v)


def quotient_with(c, s_eff_of):
    x = every(c["dtype"])
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        q = M.rn(x / s_eff_of(c["scale"], float(c["global_scale"])), "f32")
        return q if c["zero_point"] is None else M.rn(q + c["zero_point"], "f32")


MUTANTS = {
    "2.5 rounds up": lambda c: ladder(quotients(c), down=(0.25, 1.25, 5.0)),
    "5.0 rounds up": lambda c: ladder(quotients(c), down=(0.25, 1.25, 2.5)),
    "0.75 rounds down": lambda c: ladder(quotients(c), down=(0.25, 0.75, 1.25, 2.5, 5.0)),
    "-0.0 kept for x = -0.0": lambda c: ladder(quotients(c), keep_negative_zero=True),
    "s_eff not rounded to float32": lambda c: ladder(quotient_with(c, lambda s, gs: np.float64(s) / gs)) if c["kind"] == "nvfp4_quantize" else None,
    "scale * (1 / gs)": lambda c: ladder(quotient_with(c, lambda s, gs: M.rn(s * M.rn(1.0 / gs, "f32"), "f32"))) if c["kind"] == "nvfp4_quantize" else None,
}


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_the_golden_rejects_a_mutated_rounding(mutant):
    assert all(packed_mismatches(ladder(quotients(c)), c) == 0 for c in of("nvfp4_quantize")[:2]), "the restated ladder must agree"
    bad = 0
    for c in of("nvfp4_quantize") + of("mxfp4_quantize"):
        v = MUTANTS[mutant](c)
        if v is not None:
            bad += packed_mismatches(v, c)
    print(f"{mutant}: {bad} bytes differ")
    assert bad > 0


def test_the_golden_rejects_swapped_nibbles():
    bad = 0
    for c in of("nvfp4_quantize") + of("mxfp4_quantize"):
        swapped = M.e2m1(quotients(c)).reshape(-1, 2)[:, ::-1].reshape(-1)
        bad += packed_mismatches(swapped, c)
    assert bad > 0


def test_the_golden_rejects_an_e8m0_decode_one_exponent_off():
    (c,) = of("decompress_mx_scale")
    off = M.rn(np.ldexp(1.0, np.arange(256) - 126), "bf16")
    assert mismatches(off, c["value"].float().numpy()) == 255                # all but 255, whose 2^128 and 2^129 are both inf
    (d,) = of("mxfp4_decompress")
    code, rows = decompress_inputs()
    assert mismatches(M.fp4_dequantize(code, M.rn(np.ldexp(1.0, rows - 126), "bf16"), None, "bf16"), d["weight"].float().numpy()) > 0
