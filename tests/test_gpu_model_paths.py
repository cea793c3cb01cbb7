"""
The paths a whole model takes, element by element against the CPU oracle:

  A. mixed multi-tensor job tables (ct_batched through ops.batched / ops.BatchedPlan): several streaming kernels, flat and 2-D
     scale addressing, partial and single-chunk tiles, unit-size fallbacks, misaligned views and empty tensors in ONE call;
  B. what those tables cover of the ring shapes and tile schedules the library launches with, and a CUDA-graph replay;
  C. the host-resident pipeline ct_host_run_many: one large CPU tensor through the per-tensor ops (chunked), a CPU-resident model
     through ops.host_batched (chunks of many tensors sharing staging slots, an error part-way) and ModelCompressor on a
     CPU-resident model.

Every table entry names the kernel it is meant to take (a kernel label, "generic" or "empty").  The number of launches a
call makes is written next to each table, derived by hand from the planner's rules in csrc/dispatch.cu (plan_one / plan_fp4 /
plan_s24): one launch per distinct kernel, one per generic tensor, none for an empty tensor.  The count is what shows that
the table really took the paths it is meant to cover.
"""
import math
import zlib
from types import SimpleNamespace

import pytest
import torch

import oracle
from compressed_tensors_b200 import _native as N
from compressed_tensors_b200 import ops
from tests.util import same, same_values

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F8 = torch.float8_e4m3fn
BF, FP16, FP32 = torch.bfloat16, torch.float16, torch.float32
BIG = (3200, 8192)   # 26.2 M elements: >= DYNAMIC_MIN_TILES_PER_SM (24) x 132 SMs x 8192 elements -> the dynamic tile schedule


# --------------------------------------------------------------------------------------------
# problem builder shared by ops 0-4
# --------------------------------------------------------------------------------------------
class S(SimpleNamespace):
    """one table entry.  strat: tensor | channel | group | group1 (one [1, C/G] row of scales) | block (g = (bh, bw));
    dt: x dtype (ops 0, 2, 4) or scale / output dtype (ops 1, 3); sdt: scale dtype when it differs from dt; odt: output dtype of
    the dequantizing ops when it differs from the scale's; q: code dtype of op 3; off_in / off_out: byte offset of the view"""

    def __init__(self, label, shape, dt, strat, g=None, bits=4, qtype="int", zp=None, sdt=None, odt=None, q=torch.int8, off_in=0, off_out=0):
        super().__init__(label=label, shape=shape, dt=dt, strat=strat, g=g, bits=bits, qtype=qtype, zp=zp, sdt=sdt or dt, odt=odt, q=q,
                         off_in=off_in, off_out=off_out)


def _args(s):
    strat = "group" if s.strat == "group1" else s.strat
    return SimpleNamespace(strategy=strat, group_size=s.g if strat == "group" else None,
                           block_structure=list(s.g) if strat == "block" else None)


def _okw(s):
    a = _args(s)
    return dict(strategy=a.strategy, group_size=a.group_size, block_structure=a.block_structure)


def _scale_shape(s):
    R, C = s.shape
    if s.strat == "block":
        return (-(-R // s.g[0]), -(-C // s.g[1]))
    if s.strat in ("tensor", "channel"):
        return (1,) if s.strat == "tensor" else (R, 1)
    return (R if s.strat == "group" else 1, C // s.g)


def _dev_view(src: torch.Tensor, off_bytes: int) -> torch.Tensor:
    """src copied into a contiguous device view that starts `off_bytes` past a 256-byte aligned allocation"""
    k = off_bytes // src.element_size()
    base = torch.empty(src.numel() + k, dtype=src.dtype, device=DEV)
    v = base[k:k + src.numel()].view(src.shape)
    v.copy_(src.to(DEV))
    return v


def _out_view(shape, dtype, off_bytes, device=DEV) -> torch.Tensor:
    """an output buffer (at a byte offset on the device), filled with a byte pattern no kernel writes by accident"""
    n = math.prod(shape)
    if device != DEV:
        return torch.full((n * torch.empty((), dtype=dtype).element_size(),), 0xA5, dtype=torch.uint8).view(dtype).view(shape)
    k = off_bytes // torch.empty((), dtype=dtype).element_size()
    base = torch.empty(n + k, dtype=dtype, device=DEV)
    base.view(torch.uint8).fill_(0xA5)
    return base[k:k + n].view(shape)


def _qrange(bits):
    return -(1 << (bits - 1)), (1 << (bits - 1)) - 1


def _data(s, g: torch.Generator, with_x=True):
    """(x, scale, zero point) on the CPU for entry s (x is None without with_x)"""
    R, C = s.shape
    ss = _scale_shape(s)
    if s.qtype == "float":
        scale = (torch.rand(ss, generator=g) + 0.5) * 0.01
    else:
        scale = (torch.rand(ss, generator=g) + 0.5) * (2.5 / (1 << (s.bits - 1)))
    scale = scale.to(s.sdt)
    zp = None
    if s.zp == torch.int8:
        lo, hi = _qrange(s.bits)
        zp = torch.randint(max(lo, -4), min(hi, 4) + 1, ss, generator=g).to(torch.int8)
    elif s.zp == F8:
        zp = (torch.randint(-2, 3, ss, generator=g).float() * 0.5).to(F8)
    if not with_x:
        return None, scale, zp
    x = (torch.randn((R, C), generator=g) * 0.5).to(s.dt)
    if x.numel() >= 4:
        x.view(-1)[:4] = torch.tensor([0.0, -0.0, 1e-6, -1e-6]).to(s.dt)
    return x, scale, zp


def _codes(s, g, bits):
    R, C = s.shape
    if s.q == F8:
        b = torch.randint(0, 256, (R, C), generator=g).to(torch.uint8)
        b[(b & 0x7F) == 0x7F] = 0x3C                                # no NaN codes
        return b.view(F8)
    lo, hi = _qrange(bits)
    return torch.randint(lo, hi + 1, (R, C), generator=g, dtype=torch.int8)


def _problem(op, s, g, device=DEV):
    """-> (problem tuple for ops.batched / ops.host_batched, expected output on the CPU, output tensor)"""
    x, scale, zp = _data(s, g)
    zdt = zp.dtype if zp is not None else None
    a = _args(s)
    put_in = (lambda t: _dev_view(t, s.off_in)) if device == DEV else (lambda t: t.contiguous())
    put = (lambda t: t.to(DEV).contiguous()) if device == DEV else (lambda t: t.contiguous())
    R, C = s.shape
    okw = _okw(s)
    if op in (N.OP_QUANTIZE_PACK, N.OP_QUANTIZE, N.OP_FAKE_QUANTIZE):
        p = ops._resolve(x, scale, zp, a, None)
        cd = torch.result_type(x, scale)
        qt = N.Q_FLOAT if s.qtype == "float" else N.Q_INT
        if op == N.OP_QUANTIZE_PACK:
            want = oracle.pack_to_int32(oracle.quantize(x, scale, zp, num_bits=s.bits, dtype=torch.int8, **okw), s.bits)
            out = _out_view(tuple(want.shape), torch.int32, s.off_out, device)
            d = ops._desc(p, x.dtype, scale.dtype, zdt, cd, torch.int8, None, qt, s.bits)
        elif op == N.OP_QUANTIZE:
            qd = F8 if s.qtype == "float" else torch.int8
            want = oracle.quantize(x, scale, zp, num_bits=s.bits, qtype=s.qtype, dtype=qd, **okw)
            out = _out_view((R, C), qd, s.off_out, device)
            d = ops._desc(p, x.dtype, scale.dtype, zdt, cd, qd, qd, qt, s.bits)
        else:
            want = oracle.fake_quantize(x, scale, zp, num_bits=s.bits, qtype=s.qtype, **okw)
            out = _out_view((R, C), want.dtype, s.off_out, device)
            d = ops._desc(p, x.dtype, scale.dtype, zdt, cd, None, want.dtype, qt, s.bits)
        src = x
    else:
        odt = s.odt or s.sdt
        q = _codes(s, g, s.bits if op == N.OP_UNPACK_DEQUANTIZE else 8)
        want = oracle.dequantize(q, scale, zp, dtype=odt, **okw)
        if want.dtype != odt:
            want = want.to(odt)                                      # (q.to(float32) * scale).to(T): the fp8 block-checkpoint form
        like = torch.empty((R, C), dtype=torch.int8, device="meta")
        p = ops._resolve(like, scale, zp, a, None)
        if op == N.OP_UNPACK_DEQUANTIZE:
            src = oracle.pack_to_int32(q, s.bits)
            d = ops._desc(p, None, scale.dtype, zdt, None, torch.int8, odt, N.Q_INT, s.bits)
        else:
            src = q
            d = ops._desc(p, None, scale.dtype, zdt, None, q.dtype, odt, N.Q_INT, 8)
        out = _out_view((R, C), odt, s.off_out, device)
    sc = put(p.scale)
    zz = put(p.zp) if p.zp is not None else None
    return (d, put_in(src), sc, zz, out), want, out


def _check(outs, wants, specs, what):
    for i, (o, w, s) in enumerate(zip(outs, wants, specs)):
        tag = f"{what}: entry {i} [{s.label}] {tuple(s.shape)} {s.strat} {str(s.dt)[6:]}"
        o = o.cpu()
        if w.dtype == F8:
            same_values(o.view(torch.uint8), w.view(torch.uint8), tag)
        else:
            same(o, w, tag)


# --------------------------------------------------------------------------------------------
# A. the mixed tables of ops 0-4.  Tile: 2048 chunks (16384 elements) for 16-bit quantize+pack, unpack+dequantize, quantize and
# dequantize, 1024 chunks (8192 elements) otherwise (the functors' TILE in csrc/ops.cuh).  A "unit" is one thread's 1, 2 or 4 chunks of 8 elements.
# --------------------------------------------------------------------------------------------
def _many(label, dt, bits=4, **kw):
    """34 more jobs of one kernel: together with the table's own entries more than 32 jobs in that group (two table blocks)"""
    return [S(label, (8 * k, 256 + 128 * (k % 3)), dt, "group", 128, bits=bits, **kw) for k in range(1, 35)]


# op 0, quantize + pack.  Kernel (x dtype, bits, zero point, unit): A1 = bf16/4/-/1, A4 = bf16/4/-/4, A4z = bf16/4/int8/4,
# B2z = fp16/8/int8/2, C1 = fp32/4/-/1, C8 = fp32/8/-/1.  6 kernels + 5 generic tensors = 11 launches.
T_QPACK = [
    S("A1", (1, 8), BF, "tensor"),                                   # 8 elements: one chunk, unit falls back to 1 chunk
    S("A4", (16, 1024), BF, "group", 128),                           # exactly one tile
    S("A4", (19, 864), BF, "channel"),                               # one tile + one unit (2052 chunks)
    S("A4", (73, 224), BF, "group1", 32),                            # one tile - one unit (2044 chunks), one row of group scales (2-D)
    S("A1", (32, 64), BF, "group", 8),                               # group of one chunk: unit = 1 chunk
    S("A4z", (128, 256), BF, "block", (64, 64), zp=torch.int8),      # blocks that divide the tensor
    S("A1", (100, 200), BF, "block", (64, 64)),                      # blocks that do not: 25 chunks a row, unit = 1 chunk
    S("B2z", (64, 512), FP16, "channel", bits=8, zp=torch.int8),
    S("C1", (48, 256), FP32, "group", 128),
    S("C1", (896, 8192), FP32, "group", 128),                        # 896 tiles: wraps the 2-stage ring, static deal (section B)
    S("C8", (40, 96), FP32, "tensor", bits=8),
    S("generic", (8, 96), BF, "tensor", bits=3),                     # 3-bit codes
    S("generic", (5, 12), BF, "tensor"),                             # ragged: cols * bits % 32 != 0
    S("generic", (16, 256), BF, "group", 128, sdt=FP32),             # x and scale dtypes differ
    S("generic", (16, 256), BF, "group", 128, off_in=2),             # input view 2 bytes past alignment
    S("generic", (16, 256), BF, "group", 128, off_out=8),            # output view 8 bytes past alignment
    S("empty", (0, 256), BF, "tensor"),
    S("A4", BIG, BF, "group", 128),                                  # dynamic schedule for the whole A4 group
] + _many("A4", BF)
L_QPACK = 11
# under stream capture the job tables go up with one-warp upload kernels, one per 32 jobs of every group with >= 2 jobs:
# A1 (3 jobs) 1, A4 (38 jobs) 2, C1 (2 jobs) 1
L_QPACK_CAPTURED = L_QPACK + 4

# op 1, unpack + dequantize (no unit grouping; the 4-bit input of a job must be a multiple of 16 bytes for the bulk copy).
# U4 = bf16/4/-, U4z = bf16/4/int8, V8z = fp16/8/int8, W4 = fp32/4/-.  4 kernels + 7 generic = 11 launches.
T_UNPACK = [
    S("generic", (1, 8), BF, "tensor"),                              # one chunk = 4 bytes of packed input: generic
    S("U4", (1, 32), BF, "tensor"),                                  # 4 chunks = 16 bytes: the smallest streamed job
    S("U4", (16, 1024), BF, "group", 128),                           # exactly one tile
    S("U4", (19, 864), BF, "channel"),                               # one tile + 4 chunks
    S("generic", (3, 5464), BF, "channel"),                          # one tile + 1 chunk: 8196 bytes, generic
    S("U4", (73, 224), BF, "group1", 32),                            # one tile - 4 chunks, 2-D scales
    S("U4", (32, 64), BF, "group", 8),
    S("U4z", (128, 256), BF, "block", (64, 64), zp=torch.int8),
    S("U4z", (100, 200), BF, "block", (64, 64), zp=torch.int8),
    S("V8z", (64, 512), FP16, "channel", bits=8, zp=torch.int8),
    S("W4", (48, 256), FP32, "group", 128),
    S("W4", (2048, 8192), FP32, "group", 128),                       # 2048 tiles: wraps the 4-stage ring, static deal (section B)
    S("generic", (8, 96), BF, "tensor", bits=3),
    S("generic", (5, 12), BF, "tensor"),
    S("generic", (16, 256), BF, "group", 128, odt=FP32),             # output dtype differs from the scale's
    S("generic", (16, 256), BF, "group", 128, off_in=8),
    S("generic", (16, 256), BF, "group", 128, off_out=2),
    S("empty", (0, 256), BF, "tensor"),
    S("U4", BIG, BF, "group", 128),
] + _many("U4", BF)
L_UNPACK = 11

# op 2, quantize (unit 2 chunks for 16-bit x).  Signature (x dtype, kind, zero point, unit, bits):
# Q1 = bf16/int/-/1/8, Q2 = bf16/int/-/2/8, Q2b4 = bits 4, Q2b3 = bits 3, Q2z / Q1z = int8 zero point, F2z8 = bf16/fp8/fp8 zp/2,
# G2 = fp16/fp8/-/2, R1 = fp32/int/-/1/8.  9 kernels + 4 generic = 13 launches.
T_QUANT = [
    S("Q1", (1, 8), BF, "tensor", bits=8),
    S("Q2", (16, 1024), BF, "group", 128, bits=8),
    S("Q2", (25, 656), BF, "channel", bits=8),                       # one tile + one unit (2050 chunks)
    S("Q2", (31, 528), BF, "group1", 16, bits=8),                    # one tile - one unit (2046 chunks)
    S("Q1", (32, 64), BF, "group", 8, bits=8),                       # unit = 1 chunk
    S("Q2b4", (32, 128), BF, "tensor", bits=4),
    S("Q2b3", (8, 96), BF, "tensor", bits=3),                        # any width streams here: only the clamp bounds change
    S("F2z8", (64, 256), BF, "tensor", bits=8, qtype="float", zp=F8),
    S("G2", (64, 256), FP16, "channel", bits=8, qtype="float"),
    S("Q2z", (128, 256), BF, "block", (64, 64), bits=8, zp=torch.int8),
    S("Q1z", (100, 200), BF, "block", (64, 64), bits=8, zp=torch.int8),
    S("R1", (48, 256), FP32, "group", 128, bits=8),
    S("generic", (5, 12), BF, "tensor", bits=8),                     # 60 elements: not whole chunks
    S("generic", (16, 256), BF, "group", 128, bits=8, sdt=FP32),
    S("generic", (16, 256), BF, "group", 128, bits=8, off_in=2),
    S("generic", (16, 256), BF, "group", 128, bits=8, off_out=8),
    S("empty", (0, 256), BF, "tensor", bits=8),
    S("Q2", BIG, BF, "group", 128, bits=8),
] + _many("Q2", BF, bits=8)
L_QUANT = 13

# op 3, dequantize (one-byte codes: a job must be an even number of chunks, 16 bytes, for the bulk copy).  D = bf16/int8 codes/-,
# Dz = int8 zero point, E8z = bf16/fp8 codes/fp8 zp, S3 = fp8 codes, float32 scale, bf16 output, H = fp16/int8, J = fp32/int8.
# 6 kernels + 7 generic = 13 launches.
T_DEQUANT = [
    S("generic", (1, 8), BF, "tensor"),                              # one chunk = 8 bytes of codes
    S("D", (1, 16), BF, "tensor"),                                   # two chunks: the smallest streamed job
    S("D", (16, 1024), BF, "group", 128),
    S("D", (25, 656), BF, "channel"),                                # one tile + 2 chunks
    S("D", (31, 528), BF, "group1", 16),                             # one tile - 2 chunks
    S("generic", (3, 5464), BF, "channel"),                          # one tile + 1 chunk
    S("generic", (23, 712), BF, "group1", 8),                        # one tile - 1 chunk
    S("Dz", (128, 256), BF, "block", (64, 64), zp=torch.int8),
    S("Dz", (100, 200), BF, "block", (64, 64), zp=torch.int8),
    S("E8z", (64, 256), BF, "tensor", zp=F8, q=F8),
    S("S3", (100, 200), FP32, "block", (64, 64), odt=BF, q=F8),
    S("H", (64, 512), FP16, "channel"),
    S("J", (48, 256), FP32, "group", 128),
    S("generic", (16, 256), BF, "group", 128, odt=FP32),
    S("generic", (5, 12), BF, "tensor"),
    S("generic", (16, 256), BF, "group", 128, off_in=8),
    S("generic", (16, 256), BF, "group", 128, off_out=2),
    S("empty", (0, 256), BF, "tensor"),
    S("D", BIG, BF, "group", 128),
] + _many("D", BF)
L_DEQUANT = 13

# op 4, fake_quantize (1024-chunk tiles).  K4 = bf16/narrow int/-/4 bits, K4z = int8 zp, K3 = 3 bits, K8 = bf16/wide int/-/8,
# L8z = fp16/int8 zp/8 bits, M = bf16/fp8/fp8 zp, P4 = fp32/4 bits.  7 kernels + 4 generic = 11 launches.
T_FAKE = [
    S("K4", (1, 8), BF, "tensor"),
    S("K4", (8, 1024), BF, "group", 128),                            # exactly one tile
    S("K4", (5, 1640), BF, "channel"),                               # one tile + one chunk
    S("K4", (11, 744), BF, "group1", 8),                             # one tile - one chunk
    S("K4z", (128, 256), BF, "block", (64, 64), zp=torch.int8),
    S("K4z", (100, 200), BF, "block", (64, 64), zp=torch.int8),
    S("K8", (32, 128), BF, "tensor", bits=8),
    S("L8z", (64, 512), FP16, "channel", bits=8, zp=torch.int8),
    S("M", (64, 256), BF, "tensor", bits=8, qtype="float", zp=F8),
    S("P4", (48, 256), FP32, "group", 128),
    S("K3", (8, 96), BF, "tensor", bits=3),
    S("generic", (5, 12), BF, "tensor"),
    S("generic", (16, 256), BF, "group", 128, sdt=FP32),
    S("generic", (16, 256), BF, "group", 128, off_in=2),
    S("generic", (16, 256), BF, "group", 128, off_out=2),
    S("empty", (0, 256), BF, "tensor"),
    S("K4", BIG, BF, "group", 128),
] + _many("K4", BF)
L_FAKE = 11

TABLES = {
    "quantize_pack": (N.OP_QUANTIZE_PACK, T_QPACK, L_QPACK),
    "unpack_dequantize": (N.OP_UNPACK_DEQUANTIZE, T_UNPACK, L_UNPACK),
    "quantize": (N.OP_QUANTIZE, T_QUANT, L_QUANT),
    "dequantize": (N.OP_DEQUANTIZE, T_DEQUANT, L_DEQUANT),
    "fake_quantize": (N.OP_FAKE_QUANTIZE, T_FAKE, L_FAKE),
}


def _build(name, seed=0):
    op, table, n_launch = TABLES[name]
    g = torch.Generator().manual_seed(1234 + seed)
    probs, wants, outs = [], [], []
    for s in table:
        pr, w, o = _problem(op, s, g)
        probs.append(pr); wants.append(w); outs.append(o)
    return SimpleNamespace(op=op, specs=table, n_launch=n_launch, probs=probs, wants=wants, outs=outs)


_BUILT = {}


def _table(name):
    """built once per module (the oracle's side of the 26 M-element entries is the slow part)"""
    if name not in _BUILT:
        _BUILT[name] = _build(name)
    return _BUILT[name]


def _reset(t):
    for o in t.outs:
        o.view(torch.uint8).fill_(0xA5)


def _run_table(t, what):
    _reset(t)
    launches = N.launch_count()
    ops.batched(t.op, t.probs)
    used = N.launch_count() - launches
    torch.cuda.synchronize()
    assert used == t.n_launch, f"{what}: {used} launches, the table is written for {t.n_launch}"
    _check(t.outs, t.wants, t.specs, what)


def test_tables_name_the_paths_they_count():
    """the launch counts written next to the tables agree with their labels (one per kernel, one per generic tensor)"""
    for name, (_, table, n) in TABLES.items():
        labels = [s.label for s in table]
        assert len(table) >= 40, name
        fast = {l for l in labels if l not in ("generic", "empty")}
        assert n == len(fast) + labels.count("generic"), name
        assert max(labels.count(l) for l in fast) > 32, f"{name}: no kernel group with more than 32 jobs"
    for labels, n in (([e[1] for e in T_FP4], L_FP4), ([e[0] for e in T_FP4D], L_FP4D)):
        assert n == len(set(labels) - {"generic", "empty"}) + labels.count("generic")


@pytest.mark.parametrize("name", list(TABLES))
def test_mixed_table_vs_oracle(name):
    _run_table(_table(name), name)


# ---- FP4 and 2:4 tables --------------------------------------------------------------------
def _nv_scale(x, gs, sdt):
    s = (x.float().unflatten(-1, (-1, 16)).abs().amax(-1) / 6.0 * gs).clamp(max=448.0).to(F8).float()
    return s.clamp_min(2.0 ** -9).to(sdt)


def _mx_scale(x, group):
    e = torch.floor(torch.log2(x.float().unflatten(-1, (-1, group)).abs().amax(-1).clamp_min(1e-20))) - 2
    return torch.exp2(e).to(x.dtype)


# op 8, quantize + pack to FP4.  NV kernels (x dtype, scale kind, zero point): N1 = bf16/bf16 scale/-, N2 = bf16/float32 scale/-,
# N2z = bf16/float32 scale/fp8 zp, O1 = fp16/fp16 scale/-.  MX (group 32 / 64, arithmetic in x's dtype): X0 = bf16/-, X2 = bf16/uint8 zp,
# Y3 = fp16/int8 zp.  Every NV tensor has its own global scale (Job.aux).  7 kernels + 3 generic = 10 launches.
# (kind, label, shape, x dtype, scale dtype, group, zero point dtype, magnitude of x)
T_FP4 = [
    ("nv", "N1", (8, 1024), BF, BF, 16, None, 1.0),                  # exactly one tile (1024 chunks)
    ("nv", "N1", (257, 32), BF, BF, 16, None, 30.0),                 # one tile + one unit (4 chunks)
    ("nv", "N1", (2, 32), BF, BF, 16, None, 0.01),                   # two units
    # one unit: a one-row tensor's [1, C/16] scale resolves to a shared row of scales (s_row_stride 0), which the FP4 kernels
    # only address generically
    ("nv", "generic", (1, 32), BF, BF, 16, None, 0.02),
    ("nv", "N1", (64, 256), BF, BF, 16, None, 3e-3),
    ("nv", "N2", (64, 512), BF, FP32, 16, None, 2.0),
    ("nv", "N2z", (32, 256), BF, FP32, 16, F8, 0.5),
    ("nv", "O1", (64, 256), FP16, FP16, 16, None, 7.0),
    ("mx", "X0", (64, 512), BF, BF, 32, None, 1.0),
    ("mx", "X0", (32, 256), BF, BF, 64, None, 0.1),
    ("mx", "X2", (64, 256), BF, BF, 32, torch.uint8, 1.0),
    ("mx", "Y3", (64, 256), FP16, FP16, 32, torch.int8, 1.0),
    ("nv", "generic", (4, 48), BF, BF, 16, None, 1.0),               # cols % 32 != 0
    ("nv", "generic", (16, 64), FP32, FP32, 16, None, 1.0),          # float32 weights
    ("nv", "empty", (0, 64), BF, BF, 16, None, 1.0),
]
L_FP4 = 10


def _fp4_problem(entry, g, device=DEV):
    kind, label, (R, C), dt, sdt, group, zdt, mag = entry
    x = (torch.randn((R, C), generator=g) * mag).to(dt)
    if x.numel() >= 2:
        x.view(-1)[:2] = torch.tensor([0.0, -0.0]).to(dt)
    if kind == "nv":
        gs = (448.0 * 6.0 / x.float().abs().amax().clamp_min(1e-6)).reshape(1) if x.numel() else torch.ones(1)
        s = _nv_scale(x, gs, sdt) if x.numel() else torch.ones((R, C // 16), dtype=sdt)
        a = SimpleNamespace(strategy="tensor_group", group_size=16, block_structure=None, num_bits=4, type="float")
    else:
        gs = None
        s = _mx_scale(x, group)
        a = SimpleNamespace(strategy="group", group_size=group, block_structure=None, num_bits=4, type="float")
    zp = None
    if zdt == F8:
        zp = (torch.randint(-2, 3, s.shape, generator=g).float() * 0.5).to(F8)
    elif zdt is not None:
        zp = torch.zeros(s.shape, dtype=zdt)
        zp.view(-1)[::7] = 1
    want = oracle.pack_fp4_to_uint8(oracle.quantize(x, s, zp, strategy=a.strategy, group_size=group, num_bits=4, qtype="float", global_scale=gs))
    scale, gsv, se = ops._global_scale(s, gs)
    cd = torch.result_type(x, scale if gsv is None else ops._like(scale, se))
    p = ops._resolve(x, scale, zp, a, None)
    d = ops._desc(p, x.dtype, p.scale.dtype, zdt, cd, x.dtype, None, N.Q_FP4, 4, se)
    put = (lambda t: t.to(DEV).contiguous()) if device == DEV else (lambda t: t.contiguous())
    keep = put(gsv) if gsv is not None else None
    if keep is not None:
        d.global_scale = keep.data_ptr()                            # device pointer for ct_batched, host pointer for ct_host_run_many
    out = _out_view((R, C // 2), torch.uint8, 0, device)
    return (d, put(x), put(p.scale), put(p.zp) if p.zp is not None else None, out), want, out, keep


# op 9, unpack + dequantize FP4 (bulk copies need n % 32 == 0).  Signatures (output dtype, scale kind): Sb = bf16/bf16 scale,
# F8b = bf16/stored fp8, E8b = bf16/stored E8M0, Sh = fp16/fp16 scale.  The kernel does not know whether a job has a
# global scale: Sb jobs of 128 tiles with and without one alternate, and the static deal hands each CTA tiles of different jobs
# (section B).  4 kernels + 1 generic = 5 launches.
# (label, shape, scale kind, output dtype, group, global scale)
T_FP4D = [("Sb", (512, 2048), "same", BF, 16, (i % 2 == 0)) for i in range(8)] + [
    ("F8b", (64, 256), "fp8", BF, 16, True),
    ("F8b", (128, 512), "fp8", BF, 16, True),
    ("E8b", (64, 256), "e8m0", BF, 32, False),
    ("Sb", (64, 256), "same", BF, 32, False),
    ("Sh", (64, 256), "same", FP16, 16, False),
    ("Sh", (32, 512), "same", FP16, 32, False),
    ("generic", (3, 16), "same", BF, 16, True),                      # 48 elements: 24 bytes of input, not a bulk-copy multiple
    ("empty", (0, 32), "same", BF, 16, True),
]
L_FP4D = 5


def _fp4d_problem(entry, g, device=DEV):
    label, (R, C), kind, odt, group, has_gs = entry
    packed = torch.randint(0, 256, (R, C // 2), generator=g).to(torch.uint8)
    sf = torch.exp2(torch.randint(-6, 3, (R, C // group), generator=g).float()) * (1 + torch.randint(0, 4, (R, C // group), generator=g).float() / 8)
    gs = (torch.rand(1, generator=g) * 100 + 1).float() if has_gs else None
    if kind == "fp8":
        stored = sf.to(F8)
        s_float, code, base = stored.to(odt), N.DT[F8], odt
    elif kind == "e8m0":
        stored = oracle.compress_mx_scale(sf.to(BF))
        s_float, code, base = oracle.decompress_mx_scale(stored), N.DT_E8M0, odt
    else:
        stored = sf.to(odt)
        s_float, code, base = stored, N.DT[odt], odt
    want = oracle.dequantize(oracle.unpack_fp4_from_uint8(packed, R, C, odt), s_float, None, strategy="group", group_size=group,
                             global_scale=gs, dtype=odt)
    se = torch.float32 if gs is not None else base
    like = torch.empty((R, C), dtype=torch.int8, device="meta")
    p = ops._resolve(like, stored, None, SimpleNamespace(strategy="group", group_size=group, block_structure=None), None)
    d = ops._desc(p, None, torch.float32, None, None, None, odt, N.Q_FP4, 4, se)
    d.scale_dtype = code
    put = (lambda t: t.to(DEV).contiguous()) if device == DEV else (lambda t: t.contiguous())
    keep = put(gs) if gs is not None else None
    if keep is not None:
        d.global_scale = keep.data_ptr()
    out = _out_view((R, C), odt, 0, device)
    return (d, put(packed), put(p.scale), None, out), want, out, keep


def _run_fp4(op, table, builder, n_launch, what):
    g = torch.Generator().manual_seed(77)
    probs, wants, outs, keep = [], [], [], []
    for e in table:
        pr, w, o, k = builder(e, g)
        probs.append(pr); wants.append(w); outs.append(o); keep.append(k)
    launches = N.launch_count()
    ops.batched(op, probs)
    used = N.launch_count() - launches
    torch.cuda.synchronize()
    assert used == n_launch, f"{what}: {used} launches, the table is written for {n_launch}"
    for i, (o, w, e) in enumerate(zip(outs, wants, table)):
        same(o.cpu(), w, f"{what}: entry {i} {e[:3]}")


def test_mixed_fp4_quantize_pack_table_vs_oracle():
    _run_fp4(N.OP_QUANTIZE_PACK_FP4, T_FP4, _fp4_problem, L_FP4, "fp4 quantize_pack")


def test_mixed_fp4_unpack_dequantize_table_vs_oracle():
    _run_fp4(N.OP_UNPACK_DEQUANTIZE_FP4, T_FP4D, _fp4d_problem, L_FP4D, "fp4 unpack_dequantize")


def test_fused_nvfp4_observer_table_vs_oracle():
    """op 10 over several tensors of very different maxima, bf16 and fp16 (one kernel each = 2 launches; the empty one none)"""
    from compressed_tensors_b200.quantization import QuantizationArgs
    from compressed_tensors_b200.quantization.utils import calculate_qparams

    g = torch.Generator().manual_seed(5)
    a = QuantizationArgs(num_bits=4, type="float", symmetric=True, strategy="tensor_group", group_size=16, scale_dtype=F8)
    shapes = [((8, 1024), BF, 1.0), ((257, 32), BF, 40.0), ((64, 256), BF, 1e-3), ((33, 1056), FP16, 3.0), ((5, 64), FP16, 0.2),
              ((0, 64), BF, 1.0)]
    probs, want, outs, keep = [], [], [], []
    for (R, C), dt, mag in shapes:
        x = (torch.randn((R, C), generator=g) * mag).to(dt)
        if R:
            x[0, :16] = 0                                                # a dead group
        gs = (448.0 * 6.0 / x.float().abs().amax().clamp_min(1e-6)).reshape(1) if R else torch.ones(1)
        if R:
            grp = x.unflatten(-1, (-1, 16))
            s, _ = calculate_qparams(grp.amin(-1), grp.amax(-1), a, global_scale=gs)
            want.append((oracle.pack_fp4_to_uint8(oracle.quantize(x, s, None, strategy="tensor_group", group_size=16, num_bits=4, qtype="float",
                                                                  global_scale=gs)), s.to(F8)))
        else:
            want.append((torch.empty((0, C // 2), dtype=torch.uint8), torch.empty((0, C // 16), dtype=F8)))
        xd, gsd = x.to(DEV), gs.to(DEV)
        sc = torch.full((R, C // 16), 0x7F, dtype=torch.uint8, device=DEV).view(F8)
        pk = torch.full((R, C // 2), 0xA5, dtype=torch.uint8, device=DEV)
        d = N.QuantDesc()
        d.rows, d.cols, d.rdiv, d.cdiv, d.s_row_stride = R, C, 1, 16, C // 16
        d.x_dtype, d.scale_dtype, d.compute_dtype = N.DT[dt], N.DT[F8], N.DT[FP32]
        d.zp_dtype, d.q_dtype, d.out_dtype, d.qtype, d.num_bits = N.DT_NONE, N.DT[dt], N.DT_NONE, N.Q_FP4, 4
        d.global_scale, d.seff_dtype, d.aux = gsd.data_ptr(), N.DT[FP32], None
        probs.append((d, xd, sc, None, pk))
        outs.append((pk, sc))
        keep.append(gsd)
    launches = N.launch_count()
    ops.batched(N.OP_OBSERVE_QUANTIZE_PACK_FP4, probs)
    assert N.launch_count() - launches == 2
    for i, ((pk, sc), (wp, ws)) in enumerate(zip(outs, want)):
        same_values(sc.cpu().view(torch.uint8), ws.view(torch.uint8), f"observer table: tensor {i} fp8 scales")
        same(pk.cpu(), wp, f"observer table: tensor {i} nibbles")


def test_sparse24_int4_table_vs_oracle():
    """ops 11 / 12 over a table of mixed strategies, zero points and dtypes.  Signatures: bf16 without / with an int8 zero point,
    fp16 without: 3 launches per direction; the empty tensor needs none"""
    from compressed_tensors_b200.utils.semi_structured_conversions import mask_creator

    g = torch.Generator().manual_seed(24)
    table = [((64, 256), BF, "group", 128, False), ((96, 2048), BF, "channel", None, True), ((64, 512), FP16, "tensor", None, False),
             ((128, 4096), BF, "group", 32, True), ((33, 1024), BF, "group", 128, False), ((512, 4096), BF, "group", 128, False),
             ((32, 256), FP16, "group", 64, False), ((16, 64), BF, "tensor", None, True), ((0, 256), BF, "tensor", None, False)]
    cprobs, dprobs, keep = [], [], []
    for (R, C), dt, strat, group, asym in table:
        w = (torch.randn((R, C), generator=g) * 0.02).to(dt)
        if R >= 64:
            w = w * mask_creator(w).to(dt)
        wf = w.float()
        if strat == "group":
            grp = wf.unflatten(-1, (-1, group))
            mn, mx = grp.amin(-1).clamp(max=0), grp.amax(-1).clamp(min=0)
        elif strat == "channel":
            mn, mx = wf.amin(-1, keepdim=True).clamp(max=0), wf.amax(-1, keepdim=True).clamp(min=0)
        else:
            mn = wf.min().clamp(max=0).reshape(1) if R else torch.zeros(1)
            mx = wf.max().clamp(min=0).reshape(1) if R else torch.ones(1)
        sc = ((mx - mn) / 15.0 if asym else torch.maximum(mn.abs(), mx.abs()) / 7.5).to(dt)
        sc[sc == 0] = torch.finfo(dt).eps
        zp = (-8 - mn / sc.float()).clamp(-8, 7).round().to(torch.int8) if asym else None
        if R:
            want_p, want_b = oracle.sparse24_quantize_pack(w, sc, zp, strategy=strat, group_size=group)
            want_d = oracle.sparse24_unpack_dequantize(want_p, want_b, sc, zp, 4, (R, C))
        else:
            want_p, want_b = torch.empty((0, C // 16), dtype=torch.int32), torch.empty((0, C // 8), dtype=torch.uint8)
            want_d = torch.empty((0, C), dtype=dt)
        a = SimpleNamespace(strategy=strat, group_size=group, block_structure=None)
        p = ops._resolve(w, sc, zp, a, None)
        wd, scd, zpd = w.to(DEV), p.scale.to(DEV).contiguous(), (p.zp.to(DEV).contiguous() if zp is not None else None)
        packed = torch.full((R, C // 16), -1, dtype=torch.int32, device=DEV)
        bm = torch.full((R, C // 8), 0xA5, dtype=torch.uint8, device=DEV)
        back = torch.full((R, C), float("nan"), dtype=dt, device=DEV)
        zdt = torch.int8 if zp is not None else None
        d = ops._desc(p, w.dtype, sc.dtype, zdt, dt, torch.int8, None, N.Q_INT, 4)
        d.aux = bm.data_ptr()
        d2 = ops._desc(p, None, sc.dtype, zdt, None, torch.int8, dt, N.Q_INT, 4)
        d2.aux = bm.data_ptr()
        cprobs.append((d, wd, scd, zpd, packed))
        dprobs.append((d2, packed, scd, zpd, back))
        keep.append((packed, bm, back, want_p, want_b, want_d))
    launches = N.launch_count()
    ops.batched(N.OP_SPARSE24_QUANTIZE_PACK, cprobs)
    assert N.launch_count() - launches == 3
    ops.batched(N.OP_SPARSE24_UNPACK_DEQUANTIZE, dprobs)
    assert N.launch_count() - launches == 6
    for i, (packed, bm, back, wp, wb, wd) in enumerate(keep):
        same_values(bm.cpu(), wb, f"2:4 table: tensor {i} {table[i][:3]} mask bytes")
        same_values(packed.cpu(), wp, f"2:4 table: tensor {i} {table[i][:3]} packed words")
        same(back.cpu(), wd, f"2:4 table: tensor {i} {table[i][:3]} dequantized")


# --------------------------------------------------------------------------------------------
# B. ring shapes and schedules
# --------------------------------------------------------------------------------------------
# The rings the library launches with (csrc/stream.cuh: ring_shape), as (tile chunks, stages, CTAs per SM) by op and element type;
# the grid is min(SMs x CTAs, tiles).  A launch of fewer than DYNAMIC_MIN_TILES_PER_SM x 1024 chunks per SM keeps the static deal
# (csrc/dispatch.cu): CTA c takes tiles c, c + grid, c + 2 grid, ...
RINGS = {
    (N.OP_QUANTIZE_PACK, BF): (2048, 3, 2),
    (N.OP_QUANTIZE_PACK, FP16): (2048, 3, 2),
    (N.OP_QUANTIZE_PACK, FP32): (1024, 2, 3),             # 4 x 3 asked for, cut to fit 200 KB of 32 KB tiles
    (N.OP_UNPACK_DEQUANTIZE, BF): (2048, 3, 2),
    (N.OP_UNPACK_DEQUANTIZE, FP16): (2048, 3, 2),
    (N.OP_UNPACK_DEQUANTIZE, FP32): (1024, 4, 3),
    (N.OP_UNPACK_DEQUANTIZE_FP4, BF): (1024, 4, 3),
}
DYNAMIC_MIN_TILES_PER_SM = 24


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _is_static(tiles, tile, sms):
    return tiles * tile < DYNAMIC_MIN_TILES_PER_SM * 1024 * sms


def test_tables_wrap_every_ring():
    """A launch of more tiles than grid x stages gives some CTA more tiles than its ring has stages, whatever the schedule: that CTA
    reuses a stage and waits on its barriers' flipped phase.  The op 0 and 1 tables (test_mixed_table_vs_oracle) have such a launch
    on every ring those ops launch with, one of them under the static deal with several tiles a CTA."""
    sms = _sms()
    for name in ("quantize_pack", "unpack_dequantize"):
        op, table, _ = TABLES[name]
        tiles, dts = {}, {}
        for s in table:
            if s.label in ("generic", "empty"):
                continue
            tile = RINGS[(op, s.dt)][0]
            tiles[s.label] = tiles.get(s.label, 0) + -(-(math.prod(s.shape) // 8) // tile)
            dts.setdefault(s.label, set()).add(s.dt)
        wrapped, static = set(), False
        for label, n in tiles.items():
            assert len(dts[label]) == 1, f"{name}: kernel {label} mixes element types"
            tile, stages, ctas = RINGS[(op, dts[label].pop())]
            grid = min(sms * ctas, n)
            if n > grid * stages:
                wrapped.add((stages, ctas))
                static = static or _is_static(n, tile, sms)
        assert wrapped == {(st, ct) for (o, _), (_, st, ct) in RINGS.items() if o == op}, f"{name}: rings wrapped {wrapped}"
        assert static, f"{name}: no statically dealt launch wraps its ring"


def test_fp4_decompress_table_crosses_jobs_under_static_deal():
    """In the Sb launch of T_FP4D, the static deal gives most CTAs consecutive tiles of one job with a global scale and one without,
    so the FP4 decompress op must rebuild its per-tensor constants (Op::tile) when the job changes, not once per CTA
    (test_mixed_fp4_unpack_dequantize_table_vs_oracle)."""
    tile, _, ctas = RINGS[(N.OP_UNPACK_DEQUANTIZE_FP4, BF)]
    sms = _sms()
    owner = []                                                           # job of every tile of the launch
    sb = [e for e in T_FP4D if e[0] == "Sb"]
    for j, (_, (R, C), *_) in enumerate(sb):
        owner += [j] * -(-(R * C // 8) // tile)
    n = len(owner)
    grid = min(sms * ctas, n)
    assert _is_static(n, tile, sms) and n > grid, (n, grid)
    crossing = sum(any(sb[owner[t]][5] != sb[owner[t + grid]][5] for t in range(c, n - grid, grid)) for c in range(grid))
    assert crossing > grid // 2, f"{crossing} of {grid} CTAs cross between jobs with and without a global scale"


def test_mixed_table_cuda_graph_replay():
    """the mixed op-0 table captured once (job tables go up with upload kernels) and replayed on new data in the same buffers"""
    t = _build("quantize_pack", seed=1)
    plan = ops.BatchedPlan(t.op, t.probs)
    side = torch.cuda.Stream(device=DEV)
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        plan.run()
        side.synchronize()
        launches = N.launch_count()
        with torch.cuda.graph(graph, stream=side):
            plan.run()
        assert N.launch_count() - launches == L_QPACK_CAPTURED
    torch.cuda.synchronize()
    # new inputs: every x negated and scaled in place, expectations recomputed on the CPU from what the buffers now hold
    wants = []
    for (d, x, sc, zp, out), s in zip(t.probs, t.specs):
        x.mul_(-1.5)
        xc, scc = x.cpu(), sc.cpu().reshape(_scale_shape(s))
        zc = zp.cpu().reshape(_scale_shape(s)) if zp is not None else None
        wants.append(oracle.pack_to_int32(oracle.quantize(xc, scc, zc, num_bits=s.bits, dtype=torch.int8, **_okw(s)), s.bits))
    _reset(t)
    graph.replay()
    torch.cuda.synchronize()
    _check(t.outs, wants, t.specs, "graph replay")


# --------------------------------------------------------------------------------------------
# C. host-resident pipelines
# --------------------------------------------------------------------------------------------
def _need_memory(gib):
    free, _ = torch.cuda.mem_get_info(0)
    if free < gib * 2 ** 30:
        pytest.skip(f"needs {gib} GB of free device memory")


# one CPU tensor through the per-tensor ops: 32 MiB chunks.  bf16 [5000, 7168] with 128-row blocks -> chunks of 2432, 2432 and
# 136 rows, the last one crossing a partial block; int8 / 8-bit packed [9650, 7168] -> 4681 rows a chunk (4736 with 128-row
# blocks), ragged last chunk.
HOST_CASES = {
    "quantize_pack": [("block", True), ("group", False), ("tensor", True)],
    "unpack_dequantize": [("channel", True), ("group1", False), ("group", True)],     # the strategy is inferred from the scale shape
    "quantize": [("channel", False), ("block", True), ("group1", True)],
    "dequantize": [("block", False), ("tensor", True), ("group", False)],
    "fake_quantize": [("group1", False), ("channel", True), ("block", True)],
}
_HOST_DATA = {}


def _host_case(name, strat, zp):
    key = (name, strat, zp)
    if key in _HOST_DATA:
        return _HOST_DATA[key]
    wide = name in ("unpack_dequantize", "dequantize")
    shape = (9650, 7168) if wide else (5000, 7168)
    g_ = {"group": 128, "group1": 64, "block": (128, 128)}.get(strat)
    bits = 8 if name in ("unpack_dequantize", "quantize", "dequantize") else 4
    s = S("host", shape, BF, strat, g_, bits=bits, zp=torch.int8 if zp else None)
    g = torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))
    x, scale, z = _data(s, g, with_x=not wide)
    a = SimpleNamespace(**vars(_args(s)), num_bits=bits, type="int", symmetric=not zp)
    okw = _okw(s)
    if name == "quantize_pack":
        src, want = x, oracle.pack_to_int32(oracle.quantize(x, scale, z, num_bits=bits, dtype=torch.int8, **okw), bits)
        call = lambda src, sc, zz: ops.quantize_pack(src, sc, zz, a)
    elif name == "quantize":
        src, want = x, oracle.quantize(x, scale, z, num_bits=bits, dtype=torch.int8, **okw)
        call = lambda src, sc, zz: ops.quantize(src, sc, zz, a, dtype=torch.int8)
    elif name == "fake_quantize":
        src, want = x, oracle.fake_quantize(x, scale, z, num_bits=bits, **okw)
        call = lambda src, sc, zz: ops.fake_quantize(src, sc, zz, a)
    else:
        q = _codes(s, g, bits)
        want = oracle.dequantize(q, scale, z, dtype=BF, **okw)
        if name == "dequantize":
            src = q
            call = lambda src, sc, zz: ops.dequantize(src, sc, zz, args=a)
        else:
            src = oracle.pack_to_int32(q, bits)
            call = lambda src, sc, zz: ops.unpack_dequantize(src, sc, zz, bits, shape)
    _HOST_DATA.clear()                                   # one case at a time: these are hundreds of MB
    _HOST_DATA[key] = (src, scale, z, want, call)
    return _HOST_DATA[key]


@pytest.mark.parametrize("pinned", [True, False], ids=["pinned", "pageable"])
@pytest.mark.parametrize("name", list(HOST_CASES))
def test_host_pipeline_vs_oracle(name, pinned):
    _need_memory(4)
    for strat, zp in HOST_CASES[name]:
        src, scale, z, want, call = _host_case(name, strat, zp)
        assert src.numel() * src.element_size() >= 64 << 20, "at least three 32 MiB chunks"
        srci = src.pin_memory() if pinned else src
        launches = N.launch_count()
        got = call(srci, scale, z)
        assert not got.is_cuda and N.launch_count() - launches >= 3, "chunked on the device"
        same(got, want, f"{name} {strat} zp={zp} {'pinned' if pinned else 'pageable'}")


# ct_host_run_many with 1 MiB chunks: every tensor spans several chunks and chunks of different tensors share the slots.
# Rows a chunk = 1 MiB / input row bytes, rounded up to the block height: e.g. bf16 [700, 1536] with 128-row blocks -> 341 -> 384 rows,
# [1333, 1000] with 96-row blocks -> 524 -> 576 rows (chunks end inside a block unless the rounding is there).
HOST_MANY_0_4 = {
    N.OP_QUANTIZE_PACK: [S("h", (700, 1536), BF, "block", (128, 128), zp=torch.int8), S("h", (1000, 2048), BF, "group", 128),
                         S("h", (600, 1024), BF, "channel", zp=torch.int8), S("h", (1, 8), BF, "tensor"), S("h", (0, 256), BF, "tensor"),
                         S("h", (300, 4096), BF, "tensor", bits=8), S("h", (513, 1024), BF, "group1", 32, zp=torch.int8),
                         S("h", (256, 2048), FP32, "group", 128), S("h", (1333, 1000), BF, "block", (96, 192))],
    N.OP_UNPACK_DEQUANTIZE: [S("h", (3000, 1536), BF, "block", (128, 128), zp=torch.int8), S("h", (2000, 2048), BF, "group", 128),
                             S("h", (1200, 1024), FP16, "channel", bits=8, zp=torch.int8), S("h", (0, 256), BF, "tensor"),
                             S("h", (4100, 1024), BF, "group1", 32), S("h", (1100, 1000), BF, "block", (96, 192), bits=8)],
    N.OP_QUANTIZE: [S("h", (700, 1536), BF, "block", (128, 128), bits=8, zp=torch.int8), S("h", (1000, 2048), BF, "group", 128, bits=8),
                    S("h", (600, 1024), FP16, "channel", bits=8, qtype="float"), S("h", (0, 256), BF, "tensor", bits=8),
                    S("h", (513, 1024), BF, "group1", 32, bits=8, zp=torch.int8), S("h", (1333, 1000), BF, "block", (96, 192), bits=8)],
    N.OP_DEQUANTIZE: [S("h", (1400, 1536), BF, "block", (128, 128), zp=torch.int8), S("h", (1500, 2048), BF, "group", 128),
                      S("h", (1200, 1024), FP16, "channel", zp=F8, q=F8), S("h", (0, 256), BF, "tensor"),
                      S("h", (1030, 1024), BF, "group1", 32, zp=torch.int8), S("h", (1100, 1000), FP32, "block", (96, 192), odt=BF, q=F8)],
    N.OP_FAKE_QUANTIZE: [S("h", (700, 1536), BF, "block", (128, 128), zp=torch.int8), S("h", (1000, 2048), BF, "group", 128),
                         S("h", (600, 1024), BF, "channel", bits=8, qtype="float", zp=F8), S("h", (0, 256), BF, "tensor"),
                         S("h", (513, 1024), FP32, "group1", 32), S("h", (1333, 1000), BF, "block", (96, 192), zp=torch.int8)],
}


HOST_SLOTS = 4   # staging slots of the pipeline (csrc/host_pipeline.cu: NSLOT)


def _host_chunks(d, src, chunk=1 << 20):
    """row chunks the pipeline cuts one table entry into, by the rule above"""
    if d.rows * d.cols == 0:
        return 0
    rpc = max(chunk // (src.numel() * src.element_size() // d.rows), 1)
    if d.rdiv != N.INF and d.rdiv > 1:
        rpc = -(-rpc // d.rdiv) * d.rdiv
    return -(-d.rows // rpc)


def test_host_batched_vs_oracle(monkeypatch):
    monkeypatch.setenv("CT_B200_HOST_CHUNK_MB", "1")
    g = torch.Generator().manual_seed(HOST_SLOTS)
    for op, table in HOST_MANY_0_4.items():
        probs, wants, outs = [], [], []
        for s in table:
            pr, w, o = _problem(op, s, g, device="cpu")
            probs.append(pr); wants.append(w); outs.append(o)
        chunks = sum(_host_chunks(pr[0], pr[1]) for pr in probs)
        assert chunks > 2 * HOST_SLOTS, f"op {op}: {chunks} chunks do not reuse every one of the {HOST_SLOTS} staging slots"
        ops.host_batched(op, probs)
        _check(outs, wants, table, f"host_batched op {op}")
    # FP4: every NVFP4 tensor carries its own global scale as a HOST pointer
    for op, table, builder in ((N.OP_QUANTIZE_PACK_FP4, [("nv", "h", (1024, 2048), BF, BF, 16, None, 1.0), ("nv", "h", (700, 1536), BF, FP32, 16, F8, 20.0),
                                                         ("mx", "h", (512, 1024), BF, BF, 32, torch.uint8, 1.0), ("nv", "h", (0, 64), BF, BF, 16, None, 1.0),
                                                         ("nv", "h", (900, 1024), FP16, FP16, 16, None, 0.01)], _fp4_problem),
                               (N.OP_UNPACK_DEQUANTIZE_FP4, [("h", (1500, 2048), "fp8", BF, 16, True), ("h", (1000, 1024), "e8m0", BF, 32, False),
                                                             ("h", (800, 2048), "same", BF, 16, False), ("h", (1200, 1024), "same", BF, 16, True),
                                                             ("h", (0, 32), "same", BF, 16, True)], _fp4d_problem)):
        probs, wants, outs, keep = [], [], [], []
        for e in table:
            pr, w, o, k = builder(e, g, device="cpu")
            probs.append(pr); wants.append(w); outs.append(o); keep.append(k)
        ops.host_batched(op, probs)
        for i, (o, w) in enumerate(zip(outs, wants)):
            same(o, w, f"host_batched op {op}, entry {i} {table[i][:3]}")


def test_host_batched_error_part_way_leaves_no_copy_in_flight(monkeypatch):
    """a table whose second entry fails the library's dtype check after the first entry's chunks are queued (pinned buffers, so
    the copies are truly asynchronous): host_batched raises only once those copies have landed, and the pipeline works after it"""
    monkeypatch.setenv("CT_B200_HOST_CHUNK_MB", "1")
    g = torch.Generator().manual_seed(12)
    s = S("h", (2000, 2048), BF, "group", 128, bits=8)
    pr, want, _ = _problem(N.OP_QUANTIZE, s, g, device="cpu")
    good = tuple(t.pin_memory() if isinstance(t, torch.Tensor) else t for t in pr)
    assert _host_chunks(good[0], good[1]) >= 2 * HOST_SLOTS
    (d, _, sc, _, out), _, _ = _problem(N.OP_QUANTIZE, S("h", (64, 256), BF, "group", 128, bits=8), g, device="cpu")
    d.x_dtype = N.DT[torch.int8]                                  # right size for the int8 input below, but not a float to quantize
    bad = (d, torch.zeros((64, 256), dtype=torch.int8).pin_memory(), sc.pin_memory(), None, out.pin_memory())
    with pytest.raises(ValueError, match="dtype must be float"):
        ops.host_batched(N.OP_QUANTIZE, [good, bad])
    same(good[4], want, "first entry, right after the error")
    good[4].view(torch.uint8).fill_(0xA5)
    ops.host_batched(N.OP_QUANTIZE, [good])
    same(good[4], want, "the same entry, called again")


@pytest.mark.parametrize("pinned", [True, False], ids=["pinned", "pageable"])
@pytest.mark.parametrize("preset", ["W4A16", "W4A16_ASYM", "FP8", "NVFP4A16"])
def test_model_compressor_cpu_model_vs_oracle(preset, pinned, monkeypatch):
    """compress_model / decompress_model on a CPU-resident model (ct_host_run_many, 1 MiB chunks) against per-tensor oracle results"""
    from compressed_tensors_b200.compressors import ModelCompressor
    from compressed_tensors_b200.quantization import QuantizationConfig, QuantizationStatus, apply_quantization_config
    from compressed_tensors_b200.quantization.utils import calculate_qparams, generate_gparam
    from compressed_tensors_b200.utils import get_direct_state_dict

    monkeypatch.setenv("CT_B200_HOST_CHUNK_MB", "1")
    torch.manual_seed(9)
    model = torch.nn.Sequential(torch.nn.Linear(2048, 2048, bias=False), torch.nn.Linear(2048, 3072, bias=False),
                                torch.nn.Linear(3072, 2048, bias=False)).to(BF)          # 8, 12 and 12 MiB of bf16 weights
    apply_quantization_config(model, QuantizationConfig(config_groups={preset: ["Linear"]}))
    want = []
    for lin in model:
        a = lin.quantization_scheme.weights
        w = lin.weight.data
        w.view(-1)[::97] = -0.0
        if a.strategy in ("group", "tensor_group"):
            grp = w.unflatten(-1, (-1, a.group_size))
            mn, mx = grp.amin(-1), grp.amax(-1)
        elif a.strategy == "channel":
            mn, mx = w.amin(-1, keepdim=True), w.amax(-1, keepdim=True)
        else:
            mn, mx = w.min().reshape(1), w.max().reshape(1)
        gs = None
        if preset == "NVFP4A16":
            gs = generate_gparam(w.min(), w.max())
            lin.weight_global_scale.data.copy_(gs)
        s, z = calculate_qparams(mn, mx, a, global_scale=gs) if gs is not None else calculate_qparams(mn, mx, a)
        lin.weight_scale.data = s.to(lin.weight_scale.dtype if preset == "NVFP4A16" else w.dtype)
        zp = None
        if hasattr(lin, "weight_zero_point"):
            lin.weight_zero_point.data = z.to(lin.weight_zero_point.dtype)
            zp = lin.weight_zero_point.data.clone()
        if hasattr(lin, "input_scale"):
            lin.input_scale.data.fill_(0.05)
        lin.quantization_status = QuantizationStatus.FROZEN
        sc = lin.weight_scale.data.clone()
        okw = dict(strategy=a.strategy, group_size=a.group_size, block_structure=a.block_structure)
        if preset == "NVFP4A16":
            q = oracle.quantize(w, sc, None, num_bits=4, qtype="float", global_scale=gs, **okw)
            s8 = sc.to(F8)
            packed = oracle.pack_fp4_to_uint8(q)
            dense = oracle.dequantize(oracle.unpack_fp4_from_uint8(packed, *w.shape, BF), s8.to(BF), None, global_scale=gs, dtype=BF, **okw)
            want.append(({"weight_packed": packed, "weight_scale": s8}, dense))
        elif preset == "FP8":
            q = oracle.quantize(w, sc, zp, num_bits=8, qtype="float", dtype=F8, **okw)
            want.append(({"weight": q, "weight_scale": sc}, oracle.dequantize(q, sc, None, **okw)))
        else:
            zq = zp if not a.symmetric else None
            q = oracle.quantize(w, sc, zq, num_bits=4, dtype=torch.int8, **okw)
            comp = {"weight_packed": oracle.pack_to_int32(q, 4), "weight_scale": sc}
            if zq is not None:
                comp["weight_zero_point"] = oracle.pack_to_int32(zq, 4, packed_dim=0)
            want.append((comp, oracle.dequantize(q, sc, zq, dtype=sc.dtype, **okw)))
    if pinned:
        for prm in model.parameters():
            prm.data = prm.data.pin_memory()
    mc = ModelCompressor.from_pretrained_model(model)
    mc.compress_model(model)
    for i, (lin, (comp, _)) in enumerate(zip(model, want)):
        sd = get_direct_state_dict(lin)
        for k, v in comp.items():
            got = sd[k]
            assert not got.is_cuda, (preset, i, k)
            if v.dtype == F8:
                same_values(got.contiguous().view(torch.uint8), v.view(torch.uint8), f"{preset} layer {i} {k}")
            else:
                same(got.contiguous(), v.contiguous(), f"{preset} layer {i} {k}")
    mc.decompress_model(model)
    for i, (lin, (_, dense)) in enumerate(zip(model, want)):
        got = lin.weight.data
        assert not got.is_cuda
        same(got, dense, f"{preset} layer {i} decompressed weight")
