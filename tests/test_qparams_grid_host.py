"""
The memoryless min-max observer rule, calculate_qparams (quantization/utils/helpers.py:50-137), for integer and FP8 schemes on
every finite (min, max) pair of bf16 and fp16, against the reference's own values (tests/golden/qparams_grid*.pt.gz):

  * the float64 model of tests/qparams_model.py equals the golden's outright values: every max |.| of the symmetric configs and
    FP8, and both ladders of the asymmetric ones;
  * the oracle's calculate_qparams reproduces every row digest of the full asymmetric grid (about 1.07e9 pairs for bf16 and 1.01e9
    for fp16 per config); a failing row is recomputed with the model and the first pair that differs is named;
  * the product's host mirror, compressed_tensors_b200.quantization.calculate_qparams, which every shape a fused kernel declines
    goes through, equals the golden on the same outright values.

The GPU sweep (tests/test_gpu_qparams_grid.py) trusts the model and the oracle on this basis, so the tests also show that the
golden reaches the places where the rule rounds differently (every count must be positive), and that it tells each of
qparams_model.MUTANTS apart from the real rule.  Two of the counts need saying:

  * A zero point is never clamped at qmin: min <= 0 makes -min / scale >= 0, so qmin - min / scale >= qmin, and rounding to T is
    monotone.  The count is of zero points that sit at qmin; the clamp at qmax is active (scale rounded down, scales that underflow
    to 0, subnormal scales).
  * fp16 scales lie in [2^-24, 65504 / 7.5], inside [2^-100, 2^100], so only bf16 has scales on the far side of 2^+-100.
"""
import concurrent.futures as cf
import os

import numpy as np
import pytest
import torch

from compressed_tensors_b200.quantization import QuantizationArgs
from compressed_tensors_b200.quantization import calculate_qparams as mirror_qparams
from oracle.qparams import calculate_qparams as oracle_qparams
from tests import qparams_model as M
from tests.golden import load

GOLDEN = load("qparams_grid")
CASES = GOLDEN["cases"]
ROWS_PER_BATCH = 256


def of(kind, dt=None, config=None):
    return [c for c in CASES if c["kind"] == kind and dt in (None, c["dtype"]) and config in (None, c["config"])]


def as_dt(bits, dt):
    return torch.from_numpy(np.ascontiguousarray(bits, dtype=np.uint16).view(np.int16)).view(M.TORCH_DT[dt])


def golden_pairs(c):
    """(min bits, max bits) of a sym or ladder case, in the order its values are stored"""
    dt = c["dtype"]
    if c["kind"] == "sym":
        mags = M.maxima_bits(dt)
        zeros = np.zeros_like(mags)
        return (mags | np.uint16(0x8000), zeros) if c["side"] == "neg" else (zeros, mags)
    if c["side"] == "max":
        mins = M.minima_bits(dt)
        return mins, np.full_like(mins, c["rung"])
    maxs = M.maxima_bits(dt)
    return np.full_like(maxs, c["rung"]), maxs


def model_of(c, mutant=None, trace=None):
    mn, mx = golden_pairs(c)
    dt = c["dtype"]
    return M.qparams(M.bits_to_float(mn, dt), M.bits_to_float(mx, dt), c["config"], dt, mutant=mutant, trace=trace)


def mismatches(c, scale, zp):
    """pairs of case c whose scale bits or zero-point byte differ from the golden"""
    s_bits = M.float_to_bits(scale, c["dtype"]) if scale.dtype != np.uint16 else scale
    return int(((s_bits != c["scale"].numpy().view(np.uint16)) | (zp.view(np.uint8) != c["zp"].numpy())).sum())


def case_id(c):
    return f"{c['dtype']}-{c['config']}-{c['side']}" + (f"-{c['rung']:04x}" if "rung" in c else "")


def args_of(config):
    qmin, qmax, symmetric, _ = M.CONFIGS[config]
    if config == "fp8_sym":
        return QuantizationArgs(num_bits=8, type="float", symmetric=True, strategy="channel")
    return QuantizationArgs(num_bits=4 if config.startswith("int4") else 8, type="int", symmetric=symmetric, strategy="channel")


OUTRIGHT = of("sym") + of("ladder")


def test_the_golden_covers_every_config_and_the_whole_grid():
    for dt in M.TORCH_DT:
        assert len(of("sym", dt)) == 2 * len(M.SYM)
        for config in M.ASYM:
            (d,) = of("digests", dt, config)
            assert d["digests"].shape == (len(M.minima_bits(dt)), 8)
            rungs = {c["rung"] for c in of("ladder", dt, config) if c["side"] == "max"}
            assert len(rungs) >= 10 and 0 in rungs


@pytest.mark.parametrize("c", OUTRIGHT, ids=case_id)
def test_model_matches_the_golden(c):
    scale, zp = model_of(c)
    assert mismatches(c, scale, zp) == 0


@pytest.mark.parametrize("c", OUTRIGHT, ids=case_id)
def test_host_mirror_matches_the_golden(c):
    """compressed_tensors_b200.quantization.calculate_qparams: the rule every declined shape runs"""
    mn, mx = golden_pairs(c)
    scale, zp = mirror_qparams(as_dt(mn, c["dtype"]), as_dt(mx, c["dtype"]), args_of(c["config"]))
    assert mismatches(c, scale.view(torch.int16).numpy().view(np.uint16), zp.view(torch.uint8).numpy()) == 0


def oracle_digests(dt, config, rows):
    """row digests of the oracle's calculate_qparams on the given min rows (bit patterns) over every max"""
    maxs = M.maxima_bits(dt)
    qmin, qmax, symmetric, _ = M.CONFIGS[config]
    mn, mx = as_dt(np.repeat(rows, len(maxs)), dt), as_dt(np.tile(maxs, len(rows)), dt)
    s, z = oracle_qparams(mn, mx, num_bits=4 if config.startswith("int4") else 8, qtype="int", symmetric=symmetric)
    s_bits = s.view(torch.int16).numpy().view(np.uint16).reshape(len(rows), -1)
    return M.digests(s_bits, z.numpy().reshape(len(rows), -1)), s_bits, z.numpy().reshape(len(rows), -1)


def first_difference(dt, config, row, s_bits, zp):
    """the first (min, max) of one row where the scale bits or zero point differ from the model, as a message"""
    maxs = M.maxima_bits(dt)
    ms, mz = M.qparams(np.full(len(maxs), M.bits_to_float(row, dt)), M.bits_to_float(maxs, dt), config, dt)
    bad = np.nonzero((M.float_to_bits(ms, dt) != s_bits) | (mz != zp))[0]
    if len(bad) == 0:
        return f"min {float(M.bits_to_float(row, dt))!r} (0x{int(row):04x}): the model agrees with the oracle here"
    j = bad[0]
    return (f"first of {len(bad)} pairs: (min, max) = ({float(M.bits_to_float(row, dt))!r}, {float(M.bits_to_float(maxs[j], dt))!r}) "
            f"(0x{int(row):04x}, 0x{int(maxs[j]):04x}): oracle scale 0x{int(s_bits[j]):04x} zp {int(zp[j])}, "
            f"model scale 0x{int(M.float_to_bits(ms[j:j + 1], dt)[0]):04x} zp {int(mz[j])}")


@pytest.mark.parametrize("config", M.ASYM)
@pytest.mark.parametrize("dt", list(M.TORCH_DT))
def test_oracle_reproduces_every_row_digest_of_the_full_grid(dt, config):
    (g,) = of("digests", dt, config)
    want = g["digests"].numpy()
    mins = M.minima_bits(dt)
    starts = range(0, len(mins), ROWS_PER_BATCH)
    with cf.ThreadPoolExecutor(max_workers=os.cpu_count() or 1) as pool:
        for i, (got, s_bits, zp) in zip(starts, pool.map(lambda i: oracle_digests(dt, config, mins[i:i + ROWS_PER_BATCH]), starts)):
            bad = np.nonzero((got != want[i:i + len(got)]).any(axis=1))[0]
            if len(bad):
                k = bad[0]
                pytest.fail(f"{dt} {config}: {len(bad)} rows of this batch differ from the golden digest; "
                            + first_difference(dt, config, mins[i + k], s_bits[k], zp[k]))


# ------------------------------------------------------------------------------------------------------------------------------
# coverage and mutations
# ------------------------------------------------------------------------------------------------------------------------------
def traced(dt, config):
    """the model's intermediates and results over every outright golden pair of one dtype and config"""
    parts = []
    for c in of("sym" if config in M.SYM else "ladder", dt, config):
        tr = {}
        scale, zp = model_of(c, trace=tr)
        mn, mx = golden_pairs(c)
        parts.append(dict(tr, scale=scale, zp=zp, lo=M.bits_to_float(mn, dt), hi=M.bits_to_float(mx, dt)))
    return {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}


def coverage(dt, config):
    t = traced(dt, config)
    qmin, qmax, symmetric, _ = M.CONFIGS[config]
    raw = t.get("raw_scale", np.where(t["scale"] == M.EPS[dt], 0.0, t["scale"]))
    tiny = 2.0 ** -14 if dt == "fp16" else 2.0 ** -126
    n = {
        "subnormal scale": int(((raw > 0) & (raw < tiny)).sum()),
        "scale 0 -> eps": int((raw == 0).sum()),
    }
    if dt == "bf16":
        n.update({
            "scale below 2^-100": int(((raw > 0) & (raw < 2.0 ** -100)).sum()),
            "scale in [2^-100, 2^100]": int(((raw >= 2.0 ** -100) & (raw <= 2.0 ** 100)).sum()),
            "scale above 2^100": int((raw > 2.0 ** 100).sum()),
        })
    if not symmetric:
        z = t["z"]
        with np.errstate(invalid="ignore"):
            tie = np.abs(z - np.floor(z) - 0.5) == 0
            n.update({
                "zero point on .5, even below": int((tie & (np.floor(z) % 2 == 0)).sum()),
                "zero point on .5, odd below": int((tie & (np.floor(z) % 2 != 0)).sum()),
                "zero point at qmin": int((z == qmin).sum()),
                "zero point clamped at qmax": int((t["z_unclamped"] > qmax).sum()),
                "max - min = inf": int(np.isinf(t["diff"]).sum()),
            })
    return n


@pytest.mark.parametrize("config", list(M.CONFIGS))
@pytest.mark.parametrize("dt", list(M.TORCH_DT))
def test_the_golden_reaches_every_rounding_edge(dt, config):
    n = coverage(dt, config)
    print(dt, config, n)
    assert all(v > 0 for v in n.values()), n


@pytest.mark.parametrize("mutant", M.MUTANTS)
def test_the_golden_rejects_a_mutated_rule(mutant):
    bad = {}
    for c in OUTRIGHT:
        scale, zp = model_of(c, mutant=mutant)
        k = f"{c['dtype']} {c['config']}"
        bad[k] = bad.get(k, 0) + mismatches(c, scale, zp)
    print(mutant, bad)
    assert sum(bad.values()) > 0
