"""
Every call site of the observer rule obs_scale_zp (csrc/observe_core.cuh) on every finite (min, max) of bf16 and fp16 that its
config depends on, bit for bit against the reference's values (tests/golden/qparams_grid*.pt.gz), the CPU oracle and the float64
model of tests/qparams_model.py, which tests/test_qparams_grid_host.py pins to the golden.  The codes or fake-quantized values of
each fused kernel are compared with the unfused kernels (ops.quantize / quantize_pack / fake_quantize) at the same qparams, and with
oracle.quantize / oracle.fake_quantize on samples.  NaN and infinite inputs are left to tests/test_gpu_nonfinite.py; an fp16 range
whose max - min overflows has an infinite scale, and its fake-quantized values are NaN, compared as NaN without their payloads.

Each group or row holds its min and max; every other element is a quotient tie of the group's own expected qparams,
T((n + 1/2 - zp) * s), clamped into [min, max], so the quantize half of each fused kernel meets round-half-to-even at every scale,
the scales outside [2^-100, 2^100] that take IEEE division included.  The positions of the two extremes rotate over the group or
row (every lane of a 2 / 4 / 8-lane group, both halves of a packed register, every cluster rank of a wide row, both extremes in one
rank included).

Pair sets: "every max" is every finite magnitude m as (-m, 0) and (0, m), for the symmetric configs and FP8; "ladders" are every
min x about 16 max rungs and every max x the same rungs negated, for the asymmetric configs; the full grid is every min x every max.

Call sites and the tests that reach them:
  fast_observe.cu:49        ops.observe_quantize_pack (group; int4 / int8, sym / asym)
                              full asymmetric grid at group 32                  test_group_observer_full_grid
                              ladders at 64 / 128 / 256, every max at 32..256   test_group_observer_ladders_and_every_max
  observe_channel.cu:56     ops.observe_quantize(strategy="channel"), narrow rows
                              every max (int8 sym, FP8), ladders (int8 asym, packed int4 sym / asym)
                                                                                test_channel_observer_narrow_rows
  observe_channel.cu:137    ct_observe_quantize_channel on rows of 16392 columns (thread-block clusters), asserting CT_OK
                              every max (int8 sym, FP8), every min x 4 max rungs (int8 asym)
                                                                                test_channel_observer_wide_rows
  observe_tensor.cu:108     ops.observe_quantize(strategy="tensor") and observe_tensor_qparams, one range per call, 2 launches
                              binade ladder, both signs, asymmetric pairs; bf16, fp16 and fp32
                                                                                test_tensor_observer_ladder
  observe_block_mx.cu:114   ops.observe_quantize(strategy="block"), FP8_BLOCK
                              every max on [2, 16] blocks, a ladder on [128, 128] blocks
                                                                                test_block_observer_every_max
  dynamic_fake.cu:68        ops.dynamic_fake_quantize, token ([1, R, C]) and group: every max, ladders; int8 sym / asym, FP8
                                                                                test_dynamic_observer_token_and_group
  dynamic_fake.cu:133       ops.dynamic_fake_quantize, tensor, one range per call
                                                                                test_dynamic_observer_tensor
  the unfused path          shapes every fused kernel declines (group 48, 36 columns, a 2-byte-offset tensor), through the
                            host mirror of calculate_qparams              test_unfused_fallback_ladders

FP8 codes of -0 quotients: a fused kernel writes 0x80 where x is negative and x / scale rounds to -0, as the reference's quantize
does without a zero point; the checkpoint converter rewrites them (entrypoints/convert/converters/quantizer.py).  The codes here
are compared with zero point None, so every byte, 0x80 included, must equal the oracle's.
"""
import ctypes
import time

import numpy as np
import pytest
import torch

import oracle
from compressed_tensors_b200 import _native as N
from compressed_tensors_b200 import ops
from compressed_tensors_b200.quantization import QuantizationArgs
from compressed_tensors_b200.quantization.utils import helpers as host_helpers
from oracle.qparams import calculate_qparams as oracle_qparams
from tests import qparams_model as M
from tests.golden import load
from tests.util import same_nan

pytestmark = pytest.mark.gpu
DEV = "cuda"
F8 = torch.float8_e4m3fn
CASES = load("qparams_grid")["cases"]
DTS = list(M.TORCH_DT)
MAX_ELEMS = 1 << 28                   # elements built per chunk


def of(kind, dt, config):
    return [c for c in CASES if c["kind"] == kind and c["dtype"] == dt and c["config"] == config]


def u16(t):
    """bit patterns of a bf16 / fp16 tensor as int32 (for comparisons on the device)"""
    return t.contiguous().view(torch.int16).to(torch.int32) & 0xFFFF


def dev_bits(bits):
    return torch.from_numpy(np.ascontiguousarray(bits, dtype=np.uint16).view(np.int16)).to(DEV).to(torch.int32) & 0xFFFF


def from_bits(b, dt):
    return b.to(torch.int16).view(M.TORCH_DT[dt])


class Pairs:
    """(min, max) bit patterns with the golden's scale bits and zero-point bytes, all on the device"""

    def __init__(self, mn, mx, scale, zp):
        self.mn, self.mx, self.scale, self.zp = mn, mx, scale, zp

    @staticmethod
    def of_cases(cases):
        mn, mx, s, z = [], [], [], []
        for c in cases:
            a, b = golden_pairs(c)
            mn.append(a)
            mx.append(b)
            s.append(c["scale"].numpy().view(np.uint16))
            z.append(c["zp"].numpy())
        return Pairs(dev_bits(np.concatenate(mn)), dev_bits(np.concatenate(mx)), dev_bits(np.concatenate(s)),
                     torch.from_numpy(np.concatenate(z)).to(DEV).to(torch.int32))

    def __len__(self):
        return len(self.mn)

    def take(self, idx):
        return Pairs(self.mn[idx], self.mx[idx], self.scale[idx], self.zp[idx])


def golden_pairs(c):
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


def every_max(dt, config):
    return Pairs.of_cases(of("sym", dt, config))


def ladders(dt, config):
    return Pairs.of_cases(of("ladder", dt, config))


def fill(mn, mx, config, dt, width, start=0):
    """[P, width] values of dt: row i holds mn[i] and mx[i] at rotated positions, and quotient ties T((n + 1/2 - zp) * s) of the
    model's qparams of (mn[i], mx[i]), clamped into [mn[i], mx[i]], everywhere else"""
    T = M.TORCH_DT[dt]
    qmin, qmax, _, _ = M.CONFIGS[config]
    P = len(mn)
    s, zp = M.qparams(mn.double(), mx.double(), config, dt)
    i = torch.arange(start, start + P, device=DEV, dtype=torch.int64)
    k = torch.arange(width, device=DEV, dtype=torch.int64)
    n = qmin + ((k[None, :] * 7 + i[:, None] * 3) % int(qmax - qmin + 1)).to(torch.float32)
    v = ((n + 0.5 - zp[:, None].to(torch.float32)) * s[:, None].to(torch.float32)).to(T)
    v = torch.clamp(v, min=mn[:, None], max=mx[:, None])
    pmin = i % width
    pmax = (pmin + 1 + (i // width) % (width - 1)) % width
    v.scatter_(1, pmin[:, None], mn[:, None])
    v.scatter_(1, pmax[:, None], mx[:, None])
    return v


def check_qparams(what, p, scale, zp, dt, config):
    """scale bits and zero-point bytes of the kernel against the expected ones of p; a failure names the first pair that differs and
    the oracle's qparams there"""
    got_s, got_z = u16(scale.reshape(-1)), zp.reshape(-1).view(torch.uint8).to(torch.int32) if zp is not None else None
    bad = got_s != p.scale
    if got_z is not None:
        bad |= got_z != p.zp
    if bool(bad.any()):
        j = int(torch.nonzero(bad)[0])
        mn, mx = from_bits(p.mn[j:j + 1], dt).cpu(), from_bits(p.mx[j:j + 1], dt).cpu()
        qmin, qmax, sym, _ = M.CONFIGS[config]
        os_, oz = oracle_qparams(mn, mx, num_bits=4 if config.startswith("int4") else 8, qtype="float" if config == "fp8_sym" else "int",
                                 symmetric=sym)
        pytest.fail(f"{what} {dt} {config}: {int(bad.sum())} of {len(p)} pairs differ; first (min, max) = ({float(mn)!r}, {float(mx)!r}): "
                    f"kernel scale 0x{int(got_s[j]):04x} zp {int(got_z[j]) if got_z is not None else None}, expected 0x{int(p.scale[j]):04x} "
                    f"zp {int(p.zp[j])}, oracle 0x{int(u16(os_)[0]):04x} zp {int(oz.view(torch.uint8)[0])}")


def check_oracle_sample(what, p, dt, config, step=997):
    """the oracle's qparams equal the golden on a strided sample of the pairs"""
    idx = torch.arange(0, len(p), step, device=DEV)
    q = p.take(idx)
    qmin, qmax, sym, _ = M.CONFIGS[config]
    s, z = oracle_qparams(from_bits(q.mn, dt).cpu(), from_bits(q.mx, dt).cpu(), num_bits=4 if config.startswith("int4") else 8,
                          qtype="float" if config == "fp8_sym" else "int", symmetric=sym)
    assert torch.equal(u16(s).to(DEV), q.scale), f"{what}: oracle scale vs golden"
    assert torch.equal(z.view(torch.uint8).to(torch.int32).to(DEV), q.zp), f"{what}: oracle zero point vs golden"


def chunks(p, width):
    step = max(1, MAX_ELEMS // width)
    for a in range(0, len(p), step):
        yield a, p.take(slice(a, a + step))


def bits_of(config):
    return 4 if config.startswith("int4") else 8


def int_args(config, strategy, **kw):
    qmin, qmax, sym, _ = M.CONFIGS[config]
    if config == "fp8_sym":
        return QuantizationArgs(num_bits=8, type="float", symmetric=True, strategy=strategy, **kw)
    return QuantizationArgs(num_bits=bits_of(config), type="int", symmetric=sym, strategy=strategy, **kw)


def report(what, n):
    print(f"\n{what}: {n} pairs compared")


def launches(fn):
    n0 = N.launch_count()
    out = fn()
    return out, N.launch_count() - n0


# ------------------------------------------------------------------------------------------------------------------------------
# fast_observe.cu: the fused group observer
# ------------------------------------------------------------------------------------------------------------------------------
GROUPS_PER_ROW = 8


def run_group(p, dt, config, group, start=0, oracle_rows=0):
    """observe_quantize_pack on the groups of p, 8 groups to a row; checks one launch and the codes against quantize_pack at the
    kernel's qparams (and against the oracle on `oracle_rows` sampled rows); returns (scale, zp) per pair"""
    P = len(p)
    pad = -P % GROUPS_PER_ROW
    mn = torch.cat([from_bits(p.mn, dt), torch.zeros(pad, dtype=M.TORCH_DT[dt], device=DEV)])
    mx = torch.cat([from_bits(p.mx, dt), torch.zeros(pad, dtype=M.TORCH_DT[dt], device=DEV)])
    x = fill(mn, mx, config, dt, group, start).reshape(-1, GROUPS_PER_ROW * group)
    args = int_args(config, "group", group_size=group)
    (packed, scale, zp), n = launches(lambda: ops.observe_quantize_pack(x, args))
    assert n == 1, "observer + quantize + pack must be one launch"
    assert torch.equal(packed, ops.quantize_pack(x, scale, zp, args)), f"group {group} {dt} {config}: codes vs quantize_pack"
    if oracle_rows:
        r = torch.linspace(0, x.shape[0] - 1, oracle_rows, device=DEV).long()
        codes = oracle.quantize(x[r].cpu(), scale[r].cpu(), None if zp is None else zp[r].cpu(), strategy="group", group_size=group,
                                num_bits=bits_of(config), dtype=torch.int8)
        assert torch.equal(oracle.pack_to_int32(codes, bits_of(config)), packed[r].cpu()), f"group {group} {dt} {config}: codes vs oracle"
    return scale.reshape(-1)[:P], (zp.reshape(-1)[:P] if zp is not None else None)


@pytest.mark.parametrize("config", M.ASYM)
@pytest.mark.parametrize("dt", DTS)
def test_group_observer_full_grid(dt, config):
    """every (min, max) of dt at group 32: row digests against the golden, every pair against the float64 model on the device"""
    (g,) = [c for c in CASES if c["kind"] == "digests" and c["dtype"] == dt and c["config"] == config]
    want = g["digests"].numpy()
    mins, maxs = M.minima_bits(dt), M.maxima_bits(dt)
    mx_row = dev_bits(maxs)
    rows_per_slice = max(1, MAX_ELEMS // (32 * len(maxs)))
    t0, groups = time.time(), 0
    for sl, i in enumerate(range(0, len(mins), rows_per_slice)):
        rows = dev_bits(mins[i:i + rows_per_slice])
        mn, mx = rows.repeat_interleave(len(maxs)), mx_row.repeat(len(rows))
        s_m, z_m = M.qparams(from_bits(mn, dt).double(), from_bits(mx, dt).double(), config, dt)
        p = Pairs(mn, mx, u16(s_m.to(M.TORCH_DT[dt])), z_m.view(torch.uint8).to(torch.int32))
        scale, zp = run_group(p, dt, config, 32, start=i * len(maxs), oracle_rows=256 if sl % 16 == 0 else 0)
        check_qparams("group 32 vs the model", p, scale, zp, dt, config)
        got = M.digests(u16(scale).to(torch.int16).cpu().numpy().view(np.uint16).reshape(len(rows), -1),
                        zp.cpu().numpy().reshape(len(rows), -1))
        bad = np.nonzero((got != want[i:i + len(rows)]).any(axis=1))[0]
        assert len(bad) == 0, f"{dt} {config}: {len(bad)} row digests differ from the golden, first min 0x{int(mins[i + bad[0]]):04x}"
        groups += len(mn)
    report(f"group 32 full grid {dt} {config}", groups)
    print(f"  ({time.time() - t0:.1f} s)")
    assert groups == len(mins) * len(maxs)


@pytest.mark.parametrize("dt", DTS)
def test_group_observer_ladders_and_every_max(dt):
    for config in M.ASYM:
        p = ladders(dt, config)
        check_oracle_sample("ladders", p, dt, config)
        for group in (64, 128, 256):
            for a, q in chunks(p, group):
                scale, zp = run_group(q, dt, config, group, start=a, oracle_rows=64)
                check_qparams(f"group {group} ladders", q, scale, zp, dt, config)
        report(f"group 64..256 ladders {dt} {config}", 3 * len(p))
    for config in ("int4_sym", "int8_sym"):
        p = every_max(dt, config)
        for group in (32, 64, 128, 256):
            for a, q in chunks(p, group):
                scale, zp = run_group(q, dt, config, group, start=a, oracle_rows=64)
                check_qparams(f"group {group} every max", q, scale, zp, dt, config)
        report(f"group 32..256 every max {dt} {config}", 4 * len(p))


# ------------------------------------------------------------------------------------------------------------------------------
# observe_channel.cu: the channel observer, one CTA per row and one cluster per wide row
# ------------------------------------------------------------------------------------------------------------------------------
def codes_of(config, pack):
    return torch.int32 if pack else (F8 if config == "fp8_sym" else torch.int8)


def check_codes(what, x, scale, zp, args, out, config, pack, strategy, oracle_rows=64):
    if pack:
        assert torch.equal(out, ops.quantize_pack(x, scale, zp, args)), f"{what}: codes vs quantize_pack"
    else:
        want = ops.quantize(x, scale, zp, args, dtype=codes_of(config, pack))
        assert torch.equal(out.view(torch.uint8), want.view(torch.uint8)), f"{what}: codes vs quantize"
    r = torch.linspace(0, x.shape[0] - 1, oracle_rows, device=DEV).long()
    sel = (lambda t: t[r].cpu()) if strategy != "tensor" else (lambda t: t.cpu())
    codes = oracle.quantize(x[r].cpu(), sel(scale), None if zp is None else sel(zp), strategy=strategy, num_bits=bits_of(config),
                            qtype="float" if config == "fp8_sym" else "int", dtype=torch.int8 if pack else codes_of(config, pack))
    if pack:
        codes = oracle.pack_to_int32(codes, bits_of(config))
    assert torch.equal(codes.view(torch.uint8), out[r].cpu().view(torch.uint8)), f"{what}: codes vs oracle"


NARROW = [("int8_sym", "every max", False), ("fp8_sym", "every max", False), ("int8_asym", "ladders", False),
          ("int4_sym", "every max", True), ("int4_asym", "ladders", True)]


@pytest.mark.parametrize("config,pairs,pack", NARROW, ids=[f"{c}-{p.replace(' ', '_')}-{'packed' if k else 'codes'}" for c, p, k in NARROW])
@pytest.mark.parametrize("dt", DTS)
def test_channel_observer_narrow_rows(dt, config, pairs, pack):
    p = every_max(dt, config) if pairs == "every max" else ladders(dt, config)
    cols = 64
    args = int_args(config, "channel")
    for a, q in chunks(p, cols):
        x = fill(from_bits(q.mn, dt), from_bits(q.mx, dt), config, dt, cols, a)
        (out, scale, zp), n = launches(lambda: ops.observe_quantize(x, args, pack=pack))
        assert n == 1
        check_qparams(f"channel {cols}", q, scale, zp, dt, config)
        check_codes(f"channel {cols} {dt} {config}", x, scale, zp, args, out, config, pack, "channel")
    report(f"channel {cols} {dt} {config} {pairs}", len(p))


def channel_direct(x, config):
    """ct_observe_quantize_channel called directly: a decline would send ops.observe_quantize to the unfused path unseen"""
    rows, cols = x.shape
    qmin, qmax, sym, _ = M.CONFIGS[config]
    qdt = codes_of(config, False)
    d = N.QuantDesc()
    d.rows, d.cols, d.rdiv, d.cdiv, d.s_row_stride = rows, cols, 1, N.INF, 1
    d.x_dtype = d.scale_dtype = d.compute_dtype = N.DT[x.dtype]
    d.zp_dtype = N.DT_NONE if sym else N.DT[torch.int8]
    d.q_dtype, d.out_dtype, d.qtype, d.num_bits = N.DT[qdt], N.DT_NONE, (N.Q_FLOAT if config == "fp8_sym" else N.Q_INT), 8
    scale = torch.empty((rows, 1), dtype=x.dtype, device=DEV)
    zp = None if sym else torch.empty((rows, 1), dtype=torch.int8, device=DEV)
    out = torch.empty((rows, cols), dtype=qdt, device=DEV)
    idx = x.device.index
    n0 = N.launch_count()
    rc = N.lib().ct_observe_quantize_channel(ctypes.byref(d), N.ptr(x), N.ptr(scale), N.ptr(zp), N.ptr(out), idx, N.stream_ptr(idx))
    assert rc == N.CT_OK and N.launch_count() - n0 == 1
    return out, scale, zp


@pytest.mark.parametrize("config", ["int8_sym", "fp8_sym", "int8_asym"])
@pytest.mark.parametrize("dt", DTS)
def test_channel_observer_wide_rows(dt, config):
    if config == "int8_asym":
        cases = [c for c in of("ladder", dt, config) if c["side"] == "max"]
        p = Pairs.of_cases([cases[k] for k in (0, len(cases) // 3, 2 * len(cases) // 3, len(cases) - 1)])
        assert len(p) == 4 * len(M.minima_bits(dt))
    else:
        p = every_max(dt, config)
    cols = 16392
    args = int_args(config, "channel")
    for a, q in chunks(p, cols):
        x = fill(from_bits(q.mn, dt), from_bits(q.mx, dt), config, dt, cols, a * 4099)
        out, scale, zp = channel_direct(x, config)
        check_qparams(f"channel {cols}", q, scale, zp, dt, config)
        check_codes(f"channel {cols} {dt} {config}", x, scale, zp, args, out, config, False, "channel", oracle_rows=8)
    report(f"channel {cols} {dt} {config}", len(p))


# ------------------------------------------------------------------------------------------------------------------------------
# observe_tensor.cu and dynamic_fake.cu:133: one range per call
# ------------------------------------------------------------------------------------------------------------------------------
def binade_ladder(dt):
    """every binade of dt (subnormals included) x {1, 1.5, the largest mantissa}, as positive bit patterns"""
    man = 7 if dt == "bf16" else 10
    top = 0xFF if dt == "bf16" else 0x1F
    out = [0, 1, (1 << (man - 1)), (1 << man) - 1]
    for e in range(1, top):
        base = e << man
        out += [base, base | (1 << (man - 1)), base | ((1 << man) - 1)]
    return np.array(sorted(set(out)), dtype=np.uint16)


def tensor_ranges(dt, config):
    """(min bits, max bits): the binade ladder both signs for symmetric configs, a 40 x 40 sample of it for asymmetric ones"""
    lad = binade_ladder(dt)
    if M.CONFIGS[config][2]:
        return np.concatenate([lad | np.uint16(0x8000), np.zeros_like(lad)]), np.concatenate([np.zeros_like(lad), lad])
    sub = lad[np.linspace(0, len(lad) - 1, 40).astype(int)]
    return np.repeat(sub | np.uint16(0x8000), len(sub)), np.tile(sub, len(sub))


def expected(mn_bits, mx_bits, dt, config):
    """oracle and model qparams of (min, max) patterns, which must agree: (scale bits, zp bytes) as device int32"""
    qmin, qmax, sym, _ = M.CONFIGS[config]
    mn, mx = from_bits(dev_bits(mn_bits), dt).cpu(), from_bits(dev_bits(mx_bits), dt).cpu()
    s, z = oracle_qparams(mn, mx, num_bits=bits_of(config), qtype="float" if config == "fp8_sym" else "int", symmetric=sym)
    ms, mz = M.qparams(mn.double(), mx.double(), config, dt)
    assert torch.equal(s, ms.to(M.TORCH_DT[dt])) and torch.equal(z.view(torch.uint8), mz.view(torch.uint8)), "oracle vs model"
    return Pairs(dev_bits(mn_bits), dev_bits(mx_bits), u16(s).to(DEV), z.view(torch.uint8).to(torch.int32).to(DEV))


@pytest.mark.parametrize("config", ["int8_sym", "int8_asym", "fp8_sym", "int4_asym"])
@pytest.mark.parametrize("dt", DTS)
def test_tensor_observer_ladder(dt, config):
    p = expected(*tensor_ranges(dt, config), dt, config)
    x = fill(from_bits(p.mn, dt), from_bits(p.mx, dt), config, dt, 256)
    args = int_args(config, "tensor")
    pack = config == "int4_asym"
    scales, zps = [], []
    for r in range(len(p)):
        xr = x[r].reshape(8, 32).clone()
        (out, scale, zp), n = launches(lambda: ops.observe_quantize(xr, args, pack=pack))
        assert n == 2, "min / max + qparams, then the streaming quantize"
        if not pack:
            (s2, z2), n2 = launches(lambda: ops.observe_tensor_qparams(xr, args))
            assert n2 == 1 and torch.equal(s2, scale) and (z2 is None or torch.equal(z2, zp))
        if r % 64 == 0:
            check_codes(f"tensor {dt} {config}", xr, scale, zp, args, out, config, pack, "tensor", oracle_rows=8)
        scales.append(scale)
        zps.append(zp)
    check_qparams("tensor", p, torch.cat(scales), None if zps[0] is None else torch.cat(zps), dt, config)
    report(f"tensor {dt} {config}", len(p))


def test_tensor_observer_fp32_ladder():
    """fp32 on the oracle and the model, which rounds nothing but to float32 here; no golden"""
    for config in ("int8_sym", "int8_asym"):
        mn_b, mx_b = tensor_ranges("bf16", config)
        mn, mx = (torch.from_numpy((b.astype(np.uint32) << 16).view(np.float32)) for b in (mn_b, mx_b))
        want_s, want_z = oracle_qparams(mn, mx, num_bits=8, qtype="int", symmetric=M.CONFIGS[config][2])
        ms, mz = M.qparams(mn.double(), mx.double(), config, "f32")
        assert torch.equal(want_s, ms.float()) and torch.equal(want_z, mz), "oracle vs model"
        args = int_args(config, "tensor")
        got_s, got_z = [], []
        for r in range(len(mn)):
            xr = torch.stack([mn[r], mx[r], mn[r] * 0.5, mx[r] * 0.25]).repeat(4).reshape(4, 4).to(DEV)
            (out, scale, zp), n = launches(lambda: ops.observe_quantize(xr, args))
            assert n == 2
            got_s.append(scale)
            got_z.append(zp if zp is not None else torch.zeros(1, dtype=torch.int8, device=DEV))
        got_s, got_z = torch.cat(got_s).cpu(), torch.cat(got_z).cpu()
        bad = (got_s.view(torch.int32) != want_s.view(torch.int32)) | (got_z != want_z)
        assert not bool(bad.any()), f"fp32 {config}: {int(bad.sum())} ranges differ, first {int(torch.nonzero(bad)[0])}"
        report(f"tensor fp32 {config}", len(mn))


@pytest.mark.parametrize("config", ["int8_sym", "int8_asym", "fp8_sym"])
@pytest.mark.parametrize("dt", DTS)
def test_dynamic_observer_tensor(dt, config):
    p = expected(*tensor_ranges(dt, config), dt, config)
    x = fill(from_bits(p.mn, dt), from_bits(p.mx, dt), config, dt, 256)
    args = int_args(config, "tensor", dynamic=True)
    scales, zps = [], []
    for r in range(len(p)):
        xr = x[r].reshape(8, 32).clone()
        res, n = launches(lambda: ops.dynamic_fake_quantize(xr, args))
        assert res is not None and n == 2
        out, scale, zp = res
        if r % 64 == 0:
            check_fake(f"dynamic tensor {dt} {config}", xr, scale, zp, args, out, config, "tensor")
        scales.append(scale.reshape(-1))
        zps.append(zp.reshape(-1))
    check_qparams("dynamic tensor", p, torch.cat(scales), torch.cat(zps), dt, config)
    report(f"dynamic tensor {dt} {config}", len(p))


# ------------------------------------------------------------------------------------------------------------------------------
# observe_block_mx.cu: FP8_BLOCK
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTS)
def test_block_observer_every_max(dt):
    config = "fp8_sym"
    for (bh, bw), p in (((2, 16), every_max(dt, config)),
                        ((128, 128), expected(*tensor_ranges(dt, config), dt, config))):
        args = int_args(config, "block", block_structure=[bh, bw])
        for a, q in chunks(p, bh * bw):
            x = fill(from_bits(q.mn, dt), from_bits(q.mx, dt), config, dt, bh * bw, a)
            x = x.reshape(-1, bh, bw).reshape(-1, bw)                 # block i = rows [bh * i, bh * (i + 1))
            (out, scale, zp), n = launches(lambda: ops.observe_quantize(x, args))
            assert n == 1 and zp is None
            check_qparams(f"block {bh}x{bw}", q, scale, None, dt, config)
            want = ops.quantize(x, scale, None, args, dtype=F8)
            assert torch.equal(out.view(torch.uint8), want.view(torch.uint8)), f"block {bh}x{bw} {dt}: codes vs quantize"
            r = torch.arange(0, min(x.shape[0], 64 * bh), device=DEV)
            codes = oracle.quantize(x[r].cpu(), scale[: len(r) // bh].cpu(), None, strategy="block", block_structure=[bh, bw],
                                    num_bits=8, qtype="float", dtype=F8)
            assert torch.equal(codes.view(torch.uint8), out[r].cpu().view(torch.uint8)), f"block {bh}x{bw} {dt}: codes vs oracle"
        report(f"block {bh}x{bw} {dt}", len(p))


# ------------------------------------------------------------------------------------------------------------------------------
# dynamic_fake.cu:68: per-token and per-group dynamic activations
# ------------------------------------------------------------------------------------------------------------------------------
def check_fake(what, x, scale, zp, args, out, config, strategy, group=None, oracle_rows=64):
    same_nan(out, ops.fake_quantize(x, scale, zp, args), f"{what}: vs fake_quantize")
    x2 = x.reshape(-1, x.shape[-1])
    r = torch.linspace(0, x2.shape[0] - 1, oracle_rows, device=DEV).long()
    s2 = scale.reshape(x2.shape[0], -1) if strategy != "tensor" else scale.reshape(1)
    z2 = zp.reshape(x2.shape[0], -1) if strategy != "tensor" else zp.reshape(1)
    sel = (lambda t: t[r].cpu()) if strategy != "tensor" else (lambda t: t.cpu())
    o = oracle.fake_quantize(x2[r].cpu(), sel(s2), sel(z2), strategy="channel" if strategy == "token" else strategy,
                             group_size=group, num_bits=bits_of(config), qtype="float" if config == "fp8_sym" else "int")
    same_nan(out.reshape(-1, x.shape[-1])[r].cpu(), o.to(x.dtype), f"{what}: vs oracle")


DYN = [("int8_sym", "every max"), ("fp8_sym", "every max"), ("int8_asym", "ladders")]


@pytest.mark.parametrize("config,pairs", DYN, ids=[c for c, _ in DYN])
@pytest.mark.parametrize("dt", DTS)
def test_dynamic_observer_token_and_group(dt, config, pairs):
    p = every_max(dt, config) if pairs == "every max" else ladders(dt, config)
    for strategy, width in (("token", 64), ("group", 32)):
        args = int_args(config, strategy, dynamic=True, **({"group_size": 32} if strategy == "group" else {}))
        for a, q in chunks(p, width):
            pad = -len(q) % 8
            mn = torch.cat([from_bits(q.mn, dt), torch.zeros(pad, dtype=M.TORCH_DT[dt], device=DEV)])
            mx = torch.cat([from_bits(q.mx, dt), torch.zeros(pad, dtype=M.TORCH_DT[dt], device=DEV)])
            x = fill(mn, mx, config, dt, width, a)
            x = x.reshape(1, -1, width) if strategy == "token" else x.reshape(-1, 8 * width)
            res, n = launches(lambda: ops.dynamic_fake_quantize(x, args))
            assert res is not None and n == 1
            out, scale, zp = res
            check_qparams(f"dynamic {strategy}", q, scale.reshape(-1)[: len(q)], zp.reshape(-1)[: len(q)], dt, config)
            check_fake(f"dynamic {strategy} {dt} {config}", x, scale, zp, args, out, config, strategy, group=32 if strategy == "group" else None)
        report(f"dynamic {strategy} {dt} {config} {pairs}", len(p))


# ------------------------------------------------------------------------------------------------------------------------------
# the unfused path
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTS)
def test_unfused_fallback_ladders(dt, monkeypatch):
    """shapes every fused kernel declines go through the host mirror of calculate_qparams on the device: one call of it and one
    quantize launch prove the path"""
    calls = []
    real = host_helpers.calculate_qparams
    monkeypatch.setattr(host_helpers, "calculate_qparams", lambda *a, **k: calls.append(1) or real(*a, **k))
    for config in ("int8_asym", "int4_asym"):
        p = ladders(dt, config)
        # group 48: the fused group observer takes 32, 64, 128 and 256
        x = fill(from_bits(p.mn, dt), from_bits(p.mx, dt), config, dt, 48).reshape(-1, 48)
        args = int_args(config, "group", group_size=48)
        calls.clear()
        (packed, scale, zp), n = launches(lambda: ops.observe_quantize_pack(x, args))
        assert n == 1 and len(calls) == 1
        check_qparams("unfused group 48", p, scale, zp, dt, config)
        # 36 columns: the channel observer needs cols % 8 == 0
        x = fill(from_bits(p.mn, dt), from_bits(p.mx, dt), config, dt, 36)
        args = int_args(config, "channel")
        calls.clear()
        (out, scale, zp), n = launches(lambda: ops.observe_quantize(x, args))
        assert n == 1 and len(calls) == 1
        check_qparams("unfused channel 36", p, scale, zp, dt, config)
        report(f"unfused group 48 and channel 36 {dt} {config}", 2 * len(p))
    # a tensor 2 bytes off an aligned allocation: the tensor observer needs 16-byte alignment
    config = "int8_asym"
    q = expected(*tensor_ranges(dt, config), dt, config)
    x = fill(from_bits(q.mn, dt), from_bits(q.mx, dt), config, dt, 64)
    args = int_args(config, "tensor")
    scales, zps = [], []
    for r in range(len(q)):
        base = torch.empty(65, dtype=x.dtype, device=DEV)
        xr = base[1:].view(8, 8)
        xr.copy_(x[r].reshape(8, 8))
        calls.clear()
        (out, scale, zp), n = launches(lambda: ops.observe_quantize(xr, args))
        assert n == 1 and len(calls) == 1
        scales.append(scale)
        zps.append(zp)
    check_qparams("unfused tensor", q, torch.cat(scales), torch.cat(zps), dt, config)
    report(f"unfused tensor {dt} {config}", len(q))
