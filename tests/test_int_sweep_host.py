"""
The float64 model of tests/int_fp8_model.py, the CPU oracle and the library's `device = -1` CPU twins against the reference's own
outputs on every bf16 / fp16 bit pattern (tests/golden/int_sweep.pt.gz), so that the GPU sweep (tests/test_gpu_int_sweep.py) can
trust the model and the oracle where the golden stores nothing.

The sweep is only worth something if its inputs reach the places a rounding can go wrong, and if the comparison would see a wrong
rounding there.  So the tests also count, per dtype and code kind, the pre-clamp quotients that land exactly on each code's .5 tie,
on qmin - 1/2 and qmax + 1/2, on each e4m3 midpoint (subnormal ones included) and on 448 / 464 / 480, and one ulp either side of each
(every count must be positive; -128.5 is no bf16 value, so bf16 skips it), and check that the golden tells each of these mutated
models apart from the right one: ties away from zero, the zero point added in float32, clamp after round, x * (1 / s) in place of
x / s, no +-448 clamp before the e4m3 cast, round(-0.3) giving +0.0, q - zp in int8.

For integer codes "clamp after round" is the right model (qmin and qmax are integers, so the two orders agree everywhere); the
FP8 cast is where the order shows.
"""
import numpy as np
import pytest
import torch

import oracle
from compressed_tensors_b200 import ops
from tests import int_fp8_model as M
from tests.golden import load

G = load("int_sweep")
CASES, CONFIGS, SCALES = G["cases"], G["configs"], G["scales"]     # the generator's tables, stored with its outputs
CFG = {c[0]: tuple(c[1:]) for c in CONFIGS}
PATTERNS = np.arange(65536, dtype=np.uint32).astype(np.uint16)
TD = {"bf16": torch.bfloat16, "fp16": torch.float16, "f32": torch.float32}
F8 = torch.float8_e4m3fn


def of(kind):
    return [c for c in CASES if c["kind"] == kind]


def cid(c):
    return f"{c['dtype']}-{c['config']}-{c['scale']:.6g}"


def every(dt):
    with np.errstate(invalid="ignore"):
        return M.bits_to_float(PATTERNS, dt)


def x_torch(dt):
    return torch.from_numpy(PATTERNS.astype(np.int16)).view(TD[dt]).reshape(256, 256)


def mismatches(got, want):
    """bitwise float mismatches (sign of zero included), NaN matching NaN"""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    both_nan = np.isnan(got) & np.isnan(want)
    return int((((got != want) | (np.signbit(got) != np.signbit(want))) & ~both_nan).sum())


def as_float(bits, dt):
    """a golden's stored 16- / 32-bit output patterns -> float64"""
    b = bits.numpy().reshape(-1)
    if dt == "f32":
        return b.view(np.float32).astype(np.float64)
    return M.bits_to_float(b.view(np.uint16), dt)


def code_mismatches(c, rounded, keep=None):
    """codes of the golden's quantize case c that differ from the rounded values; codes of NaN quotients (those of `rounded`, or
    the `keep` mask of the right model) are not compared"""
    kind = CFG[c["config"]][0]
    keep = ~np.isnan(rounded) if keep is None else keep
    want = c["code"].numpy().reshape(-1)
    got = M.fp8_bytes(rounded) if kind == "fp8" else M.int_codes(rounded)
    return int(((got.view(want.dtype) != want) & keep).sum())


def model_rounded(c):
    kind, bits, zp = CFG[c["config"]]
    return M.quantize(every(c["dtype"]), c["scale"], c["dtype"], kind, bits, zp)


def model_fake(c):
    kind, bits, zp = CFG[c["config"]]
    return M.fake_quantize(every(c["dtype"]), c["scale"], c["dtype"], kind, bits, zp)


DQ_ROWS = np.arange(256)


def dq_inputs(config):
    """the golden's dequantize layout: row r holds every code under zero point r; (code values, zero-point values)"""
    if config == "int8_zp":
        return np.tile(DQ_ROWS - 128, (256, 1)).astype(np.float64), (DQ_ROWS - 128)[:, None].astype(np.float64)
    return np.tile(M.e4m3_decode(DQ_ROWS), (256, 1)), M.e4m3_decode(DQ_ROWS)[:, None]


def dq_torch(config):
    r = torch.arange(256, dtype=torch.int32)
    if config == "int8_zp":
        return (r - 128).to(torch.int8)[None, :].repeat(256, 1), (r - 128).to(torch.int8)[:, None]
    return r.to(torch.uint8)[None, :].repeat(256, 1).view(F8), r.to(torch.uint8)[:, None].view(F8)


# ---------------------------------------------------------------------------------------------------------------------------------
# the model, the oracle and the CPU twins against the reference's outputs
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", of("quantize"), ids=cid)
def test_model_matches_the_golden(c):
    assert code_mismatches(c, model_rounded(c)) == 0
    assert mismatches(model_fake(c), as_float(c["fake"], c["dtype"])) == 0


@pytest.mark.parametrize("c", of("dequantize"), ids=cid)
def test_model_dequantize_matches_the_golden(c):
    q, z = dq_inputs(c["config"])
    with np.errstate(invalid="ignore"):
        want = M.dequantize(q, c["scale"], c["dtype"], z)
    assert mismatches(want.reshape(-1), as_float(c["value"], c["dtype"])) == 0


def oracle_kw(kind, bits):
    return dict(strategy="tensor", num_bits=bits, qtype="float" if kind == "fp8" else "int")


def zp_t(kind, zp):
    if zp is None:
        return None
    return torch.tensor([zp]).to(F8) if kind == "fp8" else torch.tensor([zp], dtype=torch.int8)


def golden_code_tensor(c):
    kind = CFG[c["config"]][0]
    return c["code"].view(F8) if kind == "fp8" else c["code"]


def same_codes(got, c, what):
    """got: codes (int8 / float8_e4m3fn) for golden case c; codes of NaN quotients are not compared"""
    keep = torch.from_numpy(~np.isnan(model_rounded(c)).reshape(256, 256))
    g, w = got.reshape(256, 256), golden_code_tensor(c)
    if g.dtype == F8:
        g, w = g.view(torch.uint8), w.view(torch.uint8)
    bad = int(((g != w) & keep).sum())
    assert bad == 0, f"{what}: {bad} codes differ"


def same_bits(got, want_bits, what):
    g = got.reshape(-1).view(torch.int32 if got.dtype == torch.float32 else torch.int16)
    w = want_bits.reshape(-1)
    both_nan = got.reshape(-1).isnan() & w.view(got.dtype).isnan()
    bad = int(((g != w) & ~both_nan).sum())
    assert bad == 0, f"{what}: {bad} values differ"


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_oracle_matches_the_golden(dt):
    """orc_quantize_gs / orc_fake_quantize_gs / orc_dequantize_gs on every golden case of dtype dt"""
    x = x_torch(dt)
    for c in [c for c in of("quantize") if c["dtype"] == dt]:
        kind, bits, zp = CFG[c["config"]]
        s, z = torch.tensor([c["scale"]]).to(TD[dt]), zp_t(kind, zp)
        same_codes(oracle.quantize(x, s, z, dtype=F8 if kind == "fp8" else torch.int8, **oracle_kw(kind, bits)), c, cid(c))
        same_bits(oracle.fake_quantize(x, s, z, **oracle_kw(kind, bits)), c["fake"], cid(c) + " fake")
    for c in of("dequantize"):
        q, z = dq_torch(c["config"])
        same_bits(oracle.dequantize(q, torch.full((256, 1), c["scale"]).to(TD[c["dtype"]]), z), c["value"], cid(c))


class Args:
    def __init__(self, kind, bits, zp, strategy="tensor", group_size=None):
        self.strategy, self.group_size, self.block_structure = strategy, group_size, None
        self.num_bits, self.type, self.symmetric = bits, "float" if kind == "fp8" else "int", zp is None


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_cpu_twins_match_the_golden(dt, monkeypatch):
    """ct_quantize / ct_fake_quantize / ct_dequantize with device = -1 (the eager body, forced with CT_ENFORCE_EAGER=1)"""
    monkeypatch.setenv("CT_ENFORCE_EAGER", "1")
    x = x_torch(dt)
    for c in [c for c in of("quantize") if c["dtype"] == dt]:
        kind, bits, zp = CFG[c["config"]]
        s, z, a = torch.tensor([c["scale"]]).to(TD[dt]), zp_t(kind, zp), Args(kind, bits, zp)
        same_codes(ops.quantize(x, s, z, a, dtype=F8 if kind == "fp8" else torch.int8), c, cid(c) + " twin")
        same_bits(ops.fake_quantize(x, s, z, a), c["fake"], cid(c) + " twin fake")
    for c in of("dequantize"):
        q, z = dq_torch(c["config"])
        same_bits(ops.dequantize(q, torch.full((256, 1), c["scale"]).to(TD[c["dtype"]]), z), c["value"], cid(c) + " twin")


def test_the_golden_holds_every_config_and_scale():
    for dt in ("bf16", "fp16"):
        got = {(c["config"], c["scale"]) for c in of("quantize") if c["dtype"] == dt}
        assert len(got) == len(CONFIGS) * len(SCALES[dt])
    assert len(of("dequantize")) == 2 * sum(len(v) for v in SCALES.values())
    bf = {c["scale"] for c in of("quantize") if c["dtype"] == "bf16"}
    for e in (-100, 100):
        assert any(abs(s) < 2.0 ** e for s in bf) and any(abs(s) > 2.0 ** e for s in bf)
        assert any(2.0 ** (e - 1) < abs(s) < 2.0 ** (e + 1) and abs(s) < 2.0 ** e for s in bf)
    assert any(s < 0 for s in bf)


def test_pack_model_matches_the_oracle():
    """pack_to_int32 as sums of (code + 2^(B-1)) << pos against orc_pack_int32, every width 1-8 on row lengths that spill"""
    g = np.random.default_rng(7)
    for bits in range(1, 9):
        for cols in (1, 7, 32, 33, 100):
            v = g.integers(-(1 << (bits - 1)), 1 << (bits - 1), (3, cols)).astype(np.int8)
            np.testing.assert_array_equal(M.pack_int32(v, bits), oracle.pack_to_int32(torch.from_numpy(v), bits).numpy())


# ---------------------------------------------------------------------------------------------------------------------------------
# coverage and sensitivity
# ---------------------------------------------------------------------------------------------------------------------------------
def next_down_up(t, dt):
    """(t one ulp below, t one ulp above) in dt, or None when t is no dt value"""
    if float(M.rn(t, dt)) != t:
        return None
    if dt == "fp16":
        f = np.float16(t)
        return float(np.nextafter(f, np.float16(-np.inf))), float(np.nextafter(f, np.float16(np.inf)))
    b = int(np.float32(abs(t)).view(np.uint32)) >> 16
    lo, hi = float(M.bits_to_float(b - 1, "bf16")), float(M.bits_to_float(b + 1, "bf16"))
    return (lo, hi) if t > 0 else (-hi, -lo)


def edges(kind, bits):
    lo, hi = M.q_range(kind, bits)
    if kind == "int":
        return [k + 0.5 for k in range(int(lo), int(hi))] + [lo - 0.5, hi + 0.5]
    grid = M.e4m3_decode(np.arange(127))
    mids = (grid[:-1] + grid[1:]) / 2
    return sorted(set(mids.tolist() + (-mids).tolist() + [448.0, 464.0, 480.0, -448.0, -464.0, -480.0]))


def pre_clamp(c):
    kind, bits, zp = CFG[c["config"]]
    return M.add_zp(M.quotient(every(c["dtype"]), c["scale"], c["dtype"]), zp, c["dtype"])


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("family", ["int4", "int8", "int3", "int6", "fp8"])
def test_the_golden_reaches_every_edge_and_its_neighbours(dt, family):
    kind, bits, _ = CFG[family]
    cs = [c for c in of("quantize") if c["dtype"] == dt and (c["config"] == family or c["config"].startswith(family + "_"))]
    q = np.concatenate([pre_clamp(c) for c in cs])
    counts, skipped = {}, []
    for t in edges(kind, bits):
        nb = next_down_up(t, dt)
        if nb is None:
            skipped.append(t)
            continue
        for name, v in (("below", nb[0]), ("on", t), ("above", nb[1])):
            counts[(t, name)] = int((q == v).sum())
    print(f"{family} {dt}: {q.size} quotients, {len(counts)} edge points, min count {min(counts.values())}; not {dt} values: {skipped}")
    assert skipped == ([-128.5] if (dt, bits, kind) == ("bf16", 8, "int") else [])
    assert min(counts.values()) > 0, {k: n for k, n in counts.items() if n == 0}


def mutated_rounded(c, *, away=False, zp_f32=False, clamp_after=False, recip=False, no_clamp=False):
    kind, bits, zp = CFG[c["config"]]
    dt = c["dtype"]
    x, s = every(dt), c["scale"]
    lo, hi = M.q_range(kind, bits)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        q = M.rn(x * M.rn(1.0 / s, "f32"), "f32") if recip else M.rn(x / s, "f32")
        t = M.op(q + zp, dt) if (zp_f32 and zp is not None) else M.add_zp(M.rn(q, dt), zp, dt)
    if kind == "int":
        r = (lambda v: np.where(np.isnan(v), v, np.sign(v) * np.floor(np.abs(v) + 0.5))) if away else np.round
    else:
        r = lambda v: M.e4m3_decode(M.e4m3_cast(v))        # noqa: E731
    if no_clamp:
        return r(t)
    return M.clamp(r(t), lo, hi) if clamp_after else r(M.clamp(t, lo, hi))


QUANT_MUTANTS = {
    "ties away from zero": dict(away=True),
    "zero point added in float32": dict(zp_f32=True),
    "clamp after round": dict(clamp_after=True),
    "x * (1 / s)": dict(recip=True),
    "no +-448 clamp": dict(no_clamp=True),
}


@pytest.mark.parametrize("mutant", list(QUANT_MUTANTS))
def test_the_golden_rejects_a_mutated_quantize(mutant):
    cs = of("quantize")
    assert all(code_mismatches(c, mutated_rounded(c)) == 0 for c in cs[:20]), "the restated model must agree"
    bad = 0
    for c in cs:
        bad += code_mismatches(c, mutated_rounded(c, **QUANT_MUTANTS[mutant]), keep=~np.isnan(model_rounded(c)))
    print(f"{mutant}: {bad} codes differ")
    assert bad > 0


def test_the_golden_rejects_a_lost_negative_zero():
    """round(-0.3) = -0.0 shows in fake_quantize: (-0.0 - zp) * s keeps the sign when there is no zero point"""
    bad = 0
    for c in of("quantize"):
        kind, bits, zp = CFG[c["config"]]
        r = model_rounded(c)
        r = np.where(r == 0, 0.0, r)
        bad += mismatches(M.dequantize(r, c["scale"], c["dtype"], zp), as_float(c["fake"], c["dtype"]))
    print(f"round(-0.3) = +0.0: {bad} values differ")
    assert bad > 0


def test_the_golden_rejects_q_minus_zp_in_int8():
    (c,) = [c for c in of("dequantize") if c["dtype"] == "bf16" and c["config"] == "int8_zp" and c["scale"] == 1.0]
    q, z = dq_inputs("int8_zp")
    wrapped = ((q - z + 128) % 256) - 128                      # int8 arithmetic wraps
    bad = mismatches(M.op(wrapped * c["scale"], "bf16").reshape(-1), as_float(c["value"], "bf16"))
    print(f"q - zp in int8: {bad} values differ")
    assert bad > 0
