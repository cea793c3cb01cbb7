"""
Write fences around the `device = -1` CPU twins (csrc/cpu_twin.cu), and the fence helpers the GPU file shares
(tests/test_gpu_write_fences.py).

Element-by-element comparisons with the oracle cannot see two kinds of error: a store past the end of an output, which lands in the
allocator's rounding slack or in a neighbouring tensor nobody reads again, and an output element that is never written, whose stale bytes
from an identical earlier call may still be right.  Here every buffer an entry point touches is cut from a larger one:

  * outputs sit G = 64 KiB (more than one 32 KiB ring tile) after the start of a buffer filled with a poison byte and G before its end.
    Each case runs twice, with poison 0xA5 and then 0x5A: the guards must still hold the poison, the two runs must give the same output
    bytes (an element never written keeps the poison, which differs between the runs) and those bytes must be the oracle's.
  * inputs sit in the same kind of buffer, whose guards hold a value that changes the result if it is read: NaN in the first run and the
    largest finite value in the second (0x77 for integer codes, packed words and mask bytes).  Every input byte, guards included, must be
    unchanged after the call.

A failure names the entry point, the case and the byte offset.  Over-reads that neither fault nor change a result -- a vector load past
the end whose extra lanes are discarded -- cannot be seen this way and are not looked for.

This file covers the CPU twins: pack / unpack, quantize, dequantize, fake_quantize, quantize + pack, unpack + dequantize and the
Walsh-Hadamard transform, called through the library with host buffers and device = CT_DEVICE_CPU.  It needs no GPU.
"""
from __future__ import annotations

import ctypes
import math
from types import SimpleNamespace

import pytest
import torch

import oracle
from compressed_tensors_b200 import _native as N
from compressed_tensors_b200 import ops

G = 64 << 10                      # guard band on each side of every fenced view
POISONS = (0xA5, 0x5A)            # output fill of the first and the second run
CPU = -1                          # CT_DEVICE_CPU

# guard fill of an input in the two runs: a NaN, then the largest finite value, in the input's own encoding
_IN_GUARD = {
    torch.bfloat16: (b"\xc0\x7f", b"\x7f\x7f"),
    torch.float16: (b"\x00\x7e", b"\xff\x7b"),
    torch.float32: (b"\x00\x00\xc0\x7f", b"\xff\xff\x7f\x7f"),
    torch.float64: (b"\x00\x00\x00\x00\x00\x00\xf8\x7f", b"\xff\xff\xff\xff\xff\xff\xef\x7f"),
    torch.float8_e4m3fn: (b"\x7f", b"\x7e"),
}


def in_guard(dtype: torch.dtype, run: int) -> bytes:
    """the guard fill of an input of `dtype` in run 0 or 1; 0x77 for integer codes, packed words and mask bytes"""
    return _IN_GUARD[dtype][run] if dtype in _IN_GUARD else b"\x77"


def _fill(raw: torch.Tensor, pattern: bytes) -> None:
    k = len(pattern)
    raw.view(-1, k).copy_(torch.tensor(list(pattern), dtype=torch.uint8).expand(raw.numel() // k, k))


def _first_bad(region: torch.Tensor, pattern: bytes):
    """index of the first byte of `region` (which starts on a pattern boundary) that differs from the repeated pattern, or None"""
    k = len(pattern)
    want = torch.tensor(list(pattern), dtype=torch.uint8, device=region.device).repeat(region.numel() // k)
    bad = (region != want).nonzero()
    return None if bad.numel() == 0 else int(bad[0])


def _sync(t: torch.Tensor) -> None:
    if t.is_cuda:
        torch.cuda.synchronize(t.device)


class Fence:
    """one buffer of G + offset + nbytes + G bytes (rounded up to the fill pattern) filled with `fill`; `view` is the tensor at
    G + offset.  `label` names it in failure messages."""

    def __init__(self, label: str, shape, dtype: torch.dtype, offset: int, fill: bytes, device="cpu", pin: bool = False):
        self.label, self.fill = label, fill
        esize = torch.empty((), dtype=dtype).element_size()
        numel = math.prod(shape)
        self.nbytes = numel * esize
        k = len(fill)
        assert G % k == 0 and offset % k == 0 and offset % esize == 0, (label, offset, esize)
        total = G + offset + self.nbytes + G
        total += -total % k
        self.raw = torch.empty(total, dtype=torch.uint8, device=device, pin_memory=pin)
        _fill(self.raw, fill)
        self.begin = G + offset
        self.end = self.begin + self.nbytes
        self.view = self.raw[self.begin:self.end].view(dtype).view(tuple(shape))

    def guard_error(self):
        """None while every byte outside the view still holds the fill, else where the first changed byte lies"""
        _sync(self.raw)
        head = self.raw[: self.begin]
        k = len(self.fill)
        bad = _first_bad(head, self.fill)
        if bad is not None:     # report the changed byte nearest the view
            last = (head.view(-1, k) != torch.tensor(list(self.fill), dtype=torch.uint8, device=head.device)).any(1).nonzero()
            j = int(last[-1]) * k + k - 1
            return f"{self.label}: byte {j - self.begin} (before its start) changed to 0x{int(head[j]):02x}"
        tail = self.raw[self.end:]
        shift = (-self.end) % k             # the tail starts mid-pattern when nbytes is not a multiple of the pattern
        tail_pat = self.fill[k - shift:] + self.fill[: k - shift] if shift else self.fill
        bad = _first_bad(tail[: tail.numel() - tail.numel() % k], tail_pat)
        if bad is not None:
            return f"{self.label}: byte +{bad} past its end (offset {self.nbytes + bad} from its start) changed to 0x{int(tail[bad]):02x}"
        return None

    def bytes(self) -> torch.Tensor:
        _sync(self.raw)
        return self.raw[self.begin:self.end].cpu().clone()


def fenced(shape, dtype: torch.dtype, offset: int, poison: int, device="cpu", pin: bool = False, label: str = "buffer"):
    """(view, check): `view` of `shape` / `dtype` sits `offset` bytes past a 64 KiB guard inside one buffer filled with `poison`;
    check() synchronizes and asserts that every byte outside the view still holds `poison`"""
    f = Fence(label, shape, dtype, offset, bytes([poison]), device, pin)

    def check():
        err = f.guard_error()
        assert err is None, err

    return f.view, check


class FencedInput(Fence):
    """an input: `value` copied into the view of a buffer whose guards hold `fill`; unchanged() reports any byte of the whole buffer
    that the call changed"""

    def __init__(self, label: str, value: torch.Tensor, offset: int, fill: bytes, device="cpu", pin: bool = False):
        super().__init__(label, tuple(value.shape), value.dtype, offset, fill, device, pin)
        self.view.copy_(value.contiguous())
        self.snapshot = self.raw.clone()

    def changed(self):
        _sync(self.raw)
        bad = (self.raw != self.snapshot).nonzero()
        if bad.numel() == 0:
            return None
        j = int(bad[0])
        where = f"byte {j - self.begin} of the view" if self.begin <= j < self.end else (
            f"byte +{j - self.end} past its end" if j >= self.end else f"byte {j - self.begin} (before its start)")
        return f"input {self.label}: {where} was written"


def _esize(dtype: torch.dtype) -> int:
    return torch.empty((), dtype=dtype).element_size()


def _describe(b1: torch.Tensor, b2: torch.Tensor, esize: int) -> str:
    j = int((b1 != b2).nonzero()[0])
    return f"byte {j} (element {j // esize}): 0x{int(b1[j]):02x} vs 0x{int(b2[j]):02x}"


def _nan_equal(got: torch.Tensor, want: torch.Tensor):
    """index of the first element that differs bit for bit, any NaN matching any NaN; None when they match"""
    g, w = got.reshape(-1), want.reshape(-1)
    if got.dtype.is_floating_point and got.element_size() > 1 or got.dtype == torch.float8_e4m3fn:
        width = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[got.element_size()]
        both_nan = g.float().isnan() & w.float().isnan()
        bad = (g.view(width) != w.view(width)) & ~both_nan
    else:
        bad = g != w
    idx = bad.nonzero()
    return None if idx.numel() == 0 else int(idx[0])


def run_fenced(entry: str, case: str, inputs: dict, outputs: dict, call, expected: dict, *, offset: int = 256,
               in_offset=None, device="cpu", pin: bool = False, valid: dict = None, values=None):
    """Run `call(ins, outs)` twice on fenced buffers and check the guards, the inputs and the outputs.

    inputs: {name: tensor} (copied into fenced inputs on `device`); outputs: {name: (shape, dtype)}; call returns a ct_status_t.
    expected: {name: tensor or None} -- the oracle's bytes (NaN-aware), None to check writes only; valid: {name: callable(outs) ->
    number of leading elements that are defined} for outputs with a capacity tail; values: callable(outs) for a check that is not
    bit-exact.  Returns the output views of the second run."""
    in_offset = offset if in_offset is None else in_offset
    runs = []
    for run, poison in enumerate(POISONS):
        # an input keeps its own dtype's alignment (int64 permutations, fp32 scales) when the streamed tensors are misaligned
        ins = {k: FencedInput(k, v, -(-in_offset // v.element_size()) * v.element_size(), in_guard(v.dtype, run), device, pin)
               for k, v in inputs.items()}
        outs = {k: Fence(f"output {k}", s, dt, -(-offset // _esize(dt)) * _esize(dt), bytes([poison]), device, pin)
                for k, (s, dt) in outputs.items()}
        rc = call({k: f.view for k, f in ins.items()}, {k: f.view for k, f in outs.items()})
        assert rc == N.CT_OK, f"{entry}[{case}] run {run}: status {rc}: {N.last_error()}"
        errors = [e for e in [f.guard_error() for f in outs.values()] + [f.changed() for f in ins.values()] if e]
        assert not errors, f"{entry}[{case}] run {run} (poison 0x{poison:02x}): " + "; ".join(errors)
        views = {k: f.view for k, f in outs.items()}
        n_valid = {k: (valid[k](views) if valid and k in valid else None) for k in outs}
        runs.append(({k: f.bytes() for k, f in outs.items()}, views, n_valid))
    (b1, _, nv1), (b2, views, nv2) = runs
    for k, (shape, dt) in outputs.items():
        esize = torch.empty((), dtype=dt).element_size()
        assert nv1[k] == nv2[k], f"{entry}[{case}]: output {k}: {nv1[k]} vs {nv2[k]} defined elements"
        n = b1[k].numel() if nv1[k] is None else nv1[k] * esize
        if not torch.equal(b1[k][:n], b2[k][:n]):
            pytest.fail(f"{entry}[{case}]: output {k} differs between the 0xA5 and 0x5A runs (never written?) at "
                        f"{_describe(b1[k][:n], b2[k][:n], esize)}", pytrace=False)
        want = expected.get(k)
        if want is None:
            continue
        got = b2[k][:n].view(dt)
        want = want.contiguous().cpu().reshape(-1)
        assert want.dtype == dt, f"{entry}[{case}]: expected {k} is {want.dtype}, output is {dt}"
        want = want[: got.numel()]
        assert want.numel() == got.numel(), f"{entry}[{case}]: output {k}: {got.numel()} elements, oracle has {want.numel()}"
        i = _nan_equal(got, want)
        if i is not None:
            pytest.fail(f"{entry}[{case}]: output {k} element {i} (byte {i * esize}) is {got[i].item()}, the oracle's is "
                        f"{want[i].item()}", pytrace=False)
    if values is not None:
        values(views)
    return views


# --------------------------------------------------------------------------------------------------------------------------------
# problems shared with the GPU file
# --------------------------------------------------------------------------------------------------------------------------------
def qargs(strategy: str, bits: int = 4, qtype: str = "int", group_size=None, block=None):
    return SimpleNamespace(strategy=strategy, num_bits=bits, type=qtype, group_size=group_size, block_structure=block)


def scale_shape(strategy: str, rows: int, cols: int, group_size=None, block=None):
    if strategy == "tensor":
        return (1,)
    if strategy == "channel":
        return (rows, 1)
    if strategy == "group":
        return (rows, math.ceil(cols / group_size))
    return (math.ceil(rows / block[0]), math.ceil(cols / block[1]))


def qproblem(strategy, rows, cols, dtype=torch.bfloat16, bits=4, qtype="int", asym=True, group_size=None, block=None, seed=0):
    """x, scale, zero point (or None) and the args of one 2-D quantization problem whose codes span the whole range"""
    g = torch.Generator().manual_seed(seed * 7919 + rows * 31 + cols)
    x = (torch.randn(rows, cols, generator=g) * 2).to(dtype)
    ss = scale_shape(strategy, rows, cols, group_size, block)
    qmax = 448.0 if qtype == "float" else float(1 << (bits - 1))
    scale = (torch.rand(ss, generator=g) * 0.5 + 4.0 / qmax).to(dtype)
    zp = torch.randint(-(1 << (bits - 1)) // 2, (1 << (bits - 1)) // 2 + 1, ss, generator=g, dtype=torch.int8) \
        if asym and qtype == "int" else None
    return x, scale, zp, qargs(strategy, bits, qtype, group_size, block)


def oracle_kw(args) -> dict:
    return dict(strategy=args.strategy, group_size=args.group_size, block_structure=args.block_structure)


def quant_desc(op: str, x, scale, zp, args):
    """(desc, expected output) of one quantize-family op, the descriptor built by the op's own recipe in ops.py"""
    bits = int(args.num_bits)
    kw = oracle_kw(args)
    okw = dict(kw, num_bits=bits, qtype=args.type)
    q_dt = torch.float8_e4m3fn if args.type == "float" else torch.int8
    if op == "quantize":
        return ops._quantize_call(x, scale, zp, args, dtype=q_dt).desc, oracle.quantize(x, scale, zp, dtype=q_dt, **okw)
    codes = oracle.quantize(x, scale, zp, dtype=torch.int8, **okw)
    if op == "dequantize":
        c = ops._dequantize_call(codes, scale, zp, args)
        return c.desc, oracle.dequantize(codes, scale, zp, dtype=c.out_dtype, **kw).to(c.out_dtype)
    if op == "fake_quantize":
        return ops._fake_quantize_call(x, scale, zp, args).desc, oracle.fake_quantize(x, scale, zp, **okw)
    if op == "quantize_pack":
        return ops._quantize_pack_call(x, scale, zp, args).desc, oracle.pack_to_int32(codes, bits)
    assert op == "unpack_dequantize"
    # unpack_dequantize infers its strategy from the scale shape, which cannot name every block layout these problems use:
    # the same descriptor, with the problem's own args
    p = ops._resolve(x, scale, zp, args, None)
    d = ops._desc(p, None, scale.dtype, zp.dtype if zp is not None else None, None, torch.int8, scale.dtype, N.Q_INT, bits)
    return d, oracle.dequantize(codes, scale, zp, dtype=scale.dtype, **kw).to(scale.dtype)


QUANT_FNS = {"quantize": "ct_quantize", "dequantize": "ct_dequantize", "fake_quantize": "ct_fake_quantize",
             "quantize_pack": "ct_quantize_pack_int32", "unpack_dequantize": "ct_unpack_dequantize_int32"}


def quant_io(op: str, x, scale, zp, args, want):
    """(inputs, outputs) of one quantize-family op: the streamed input and the qparams, the output shape and dtype"""
    bits = int(args.num_bits)
    rows, cols = x.shape
    ins = {"scale": scale.contiguous()}
    if zp is not None:
        ins["zp"] = zp.contiguous()
    if op == "quantize_pack" or op in ("quantize", "fake_quantize"):
        ins["x"] = x
    elif op == "dequantize":
        ins["x"] = oracle.quantize(x, scale, zp, dtype=torch.int8, num_bits=bits, qtype="int", **oracle_kw(args))
    else:
        codes = oracle.quantize(x, scale, zp, dtype=torch.int8, num_bits=bits, qtype="int", **oracle_kw(args))
        ins["x"] = oracle.pack_to_int32(codes, bits)
    return ins, {"out": (tuple(want.shape), want.dtype)}


def quant_call(op: str, d, device: int, stream=None):
    fn = getattr(N.lib(), QUANT_FNS[op])
    return lambda i, o: fn(ctypes.byref(d), N.ptr(i["x"]), N.ptr(i["scale"]), N.ptr(i.get("zp")), None, N.ptr(o["out"]), device, stream)


# --------------------------------------------------------------------------------------------------------------------------------
# the CPU twins
# --------------------------------------------------------------------------------------------------------------------------------
# packed_dim 1 and 0, every width, columns and rows that leave a partial last word
PACK_SHAPES = [(1, 1), (3, 37), (5, 100), (17, 8)]


@pytest.mark.parametrize("offset", [256, 16, 4])
@pytest.mark.parametrize("packed_dim", [1, 0])
@pytest.mark.parametrize("bits", range(1, 9))
def test_cpu_pack_unpack_int32(bits, packed_dim, offset):
    lib = N.lib()
    for rows, cols in PACK_SHAPES:
        g = torch.Generator().manual_seed(bits * 100 + rows + cols)
        codes = torch.randint(-(1 << (bits - 1)), 1 << (bits - 1), (rows, cols), generator=g, dtype=torch.int8)
        packed = oracle.pack_to_int32(codes, bits, packed_dim)
        case = f"twin-bits{bits}-dim{packed_dim}-{rows}x{cols}-off{offset}"
        run_fenced("ct_pack_int32", case, {"x": codes}, {"out": (tuple(packed.shape), torch.int32)},
                   lambda i, o: lib.ct_pack_int32(N.ptr(i["x"]), N.ptr(o["out"]), rows, cols, bits, packed_dim, CPU, None),
                   {"out": packed}, offset=offset)
        run_fenced("ct_unpack_int32", case, {"x": packed}, {"out": ((rows, cols), torch.int8)},
                   lambda i, o: lib.ct_unpack_int32(N.ptr(i["x"]), N.ptr(o["out"]), rows, cols, bits, packed_dim, CPU, None),
                   {"out": codes}, offset=offset)


QUANT_CASES = [
    # (strategy, rows, cols, group_size, block, dtype, bits, qtype)
    ("tensor", 1, 13, None, None, torch.bfloat16, 8, "int"),
    ("channel", 7, 40, None, None, torch.float16, 8, "int"),
    ("group", 3, 96, 32, None, torch.bfloat16, 4, "int"),
    ("group", 1, 128, 128, None, torch.float32, 4, "int"),
    ("block", 37, 70, None, (16, 32), torch.bfloat16, 8, "int"),
    ("channel", 5, 24, None, None, torch.bfloat16, 8, "float"),
]


def _qid(c):
    s, r, col, gs, blk, dt, bits, qt = c
    return f"{s}{gs or ''}{'x'.join(map(str, blk)) if blk else ''}-{r}x{col}-{str(dt)[6:]}-{qt}{bits}"


@pytest.mark.parametrize("offset", [256, 16, 8])
@pytest.mark.parametrize("op", list(QUANT_FNS))
@pytest.mark.parametrize("c", QUANT_CASES, ids=_qid)
def test_cpu_quantize_family(c, op, offset):
    strategy, rows, cols, gs, blk, dt, bits, qt = c
    if qt == "float" and op != "quantize" and op != "fake_quantize":
        pytest.skip("fp8 codes are not packed or taken by the int8 dequantize problem built here")
    if op in ("quantize_pack", "unpack_dequantize") and bits == 8 and strategy == "block":
        bits = 4
    x, scale, zp, args = qproblem(strategy, rows, cols, dt, bits, qt, asym=(qt == "int"), group_size=gs, block=blk)
    d, want = quant_desc(op, x, scale, zp, args)
    ins, outs = quant_io(op, x, scale, zp, args, want)
    run_fenced(QUANT_FNS[op], f"twin-{_qid(c)}-off{offset}", ins, outs, quant_call(op, d, CPU), {"out": want}, offset=offset)


@pytest.mark.parametrize("offset", [256, 16, 4])
@pytest.mark.parametrize("precision", [torch.float64, torch.float32])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_cpu_hadamard_transform(dtype, precision, offset):
    from tests.test_transform_host import assert_fp64_result, assert_online_bound, structured_reference

    for log2_n, shape in ((1, (1, 1, 1, 2)), (3, (2, 1, 3, 24)), (6, (1, 2, 5, 64))):
        n = 1 << log2_n
        g = torch.Generator().manual_seed(log2_n)
        x = torch.randn(shape, generator=g).to(dtype)
        sign = torch.where(torch.rand(n, generator=g) < 0.5, -1, 1).to(torch.int8)
        perm = torch.randperm(n, generator=g)

        def call(i, o):
            j = ops._hadamard_job(i["x"], o["out"], log2_n, i["sign"], i["perm"], False, precision)
            return N.lib().ct_hadamard_transform(ctypes.byref(j), CPU, None)

        ref = structured_reference(x, n, sign, perm)
        # 16-bit inputs with float64 compute give the float64 value rounded through fp32 exactly; otherwise a bound
        exact = {"out": ref.float().to(dtype)} if precision == torch.float64 and dtype != torch.float32 else {}
        check = assert_fp64_result if precision == torch.float64 else assert_online_bound

        run_fenced("ct_hadamard_transform", f"twin-n{n}-{str(dtype)[6:]}-{str(precision)[6:]}-off{offset}",
                   {"x": x, "sign": sign, "perm": perm}, {"out": (shape, dtype)}, call, exact, offset=offset,
                   values=lambda o: check(o["out"], ref, x, n))
