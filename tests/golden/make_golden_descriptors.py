#!/usr/bin/env python
"""
Golden record of every descriptor the host front end hands to the library, captured without a GPU or the built library.

`N.lib` is replaced by a recorder that answers every `ct_*` call with CT_OK and records the entry point, its integer arguments,
every `ct_quant_desc` field (`global_scale` / `aux` as present or absent), which pointers are null (per problem for the
multi-tensor tables) and, for the call as a whole, the shape and dtype of what the public function returns or the exception it
raises.  The calls run in eager mode (`ops._mode.cpu`), so every per-tensor function builds its descriptor exactly as on the
device; the whole-model functions run on host-resident modules with a CUDA device pretended, so their `ct_host_run_many`
tables are recorded too.

    python tests/golden/make_golden_descriptors.py   ->  tests/golden/descriptors.pt.gz

`collect()` is also what tests/test_descriptor_recipes_host.py replays against the fixture.
"""
import contextlib
import ctypes
import math
import os
import sys
from types import SimpleNamespace

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from compressed_tensors_b200 import _native as N  # noqa: E402
from compressed_tensors_b200 import ops  # noqa: E402

F8 = torch.float8_e4m3fn
FLOATS = (torch.bfloat16, torch.float16, torch.float32)
_DESC_FIELDS = [name for name, _ in N.QuantDesc._fields_ if name != "_reserved"]
_TABLE_CALLS = ("ct_batched", "ct_host_run_many")


def _desc(d) -> tuple:
    return tuple((f, bool(getattr(d, f))) if f in ("global_scale", "aux") else (f, int(getattr(d, f))) for f in _DESC_FIELDS)


class Recorder:
    """stands in for the loaded library: every entry point returns CT_OK and is recorded"""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if not name.startswith("ct_"):
            raise AttributeError(name)

        def call(*args):
            self.calls.append(self._record(name, args))
            return N.CT_OK

        return call

    @staticmethod
    def _record(name, args):
        out = [name]
        n = int(args[1]) if name in _TABLE_CALLS else 0
        for i, a in enumerate(args):
            if isinstance(a, bool) or isinstance(a, int):
                out.append(("int", int(a)))
            elif a is None:
                out.append(("null",))
            elif isinstance(a, ctypes.Array) and a._type_ is N.QuantDesc:
                out.append(("descs", tuple(_desc(a[k]) for k in range(n))))
            elif isinstance(a, ctypes.c_void_p):
                if name in _TABLE_CALLS and 3 <= i <= 6:     # in / scale / zp / out pointer tables
                    table = (ctypes.c_void_p * n).from_address(a.value) if n else []
                    out.append(("table", tuple(bool(p) for p in table)))
                else:
                    out.append(("ptr", bool(a.value)))
            elif type(a).__name__ == "CArgObject":
                obj = a._obj
                out.append(("desc", _desc(obj)) if isinstance(obj, N.QuantDesc) else ("byref", type(obj).__name__))
            else:
                out.append(("arg", type(a).__name__))
        return tuple(out)


def _describe(v):
    if isinstance(v, torch.Tensor):
        return ("tensor", tuple(v.shape), str(v.dtype), v.device.type)
    if isinstance(v, (tuple, list)):
        return tuple(_describe(x) for x in v)
    if v is None:
        return None
    return ("value", repr(v))


@contextlib.contextmanager
def recording(pretend_cuda: bool = False):
    """the recorder as the library, eager mode, and (pretend_cuda) a CUDA device for the whole-model functions' host queue"""
    rec = Recorder()
    saved = (N.lib, N.stream_ptr, N.require_device, torch.cuda.is_available, getattr(ops._mode, "cpu", False))
    N.lib = lambda: rec
    N.stream_ptr = lambda idx: None
    if pretend_cuda:
        N.require_device = lambda device=None: 0
        torch.cuda.is_available = lambda: True
    ops._mode.cpu = True
    try:
        yield rec
    finally:
        N.lib, N.stream_ptr, N.require_device, torch.cuda.is_available, ops._mode.cpu = saved


def run(rec: Recorder, fn, *args, **kwargs) -> dict:
    start = len(rec.calls)
    try:
        result = ("ok", _describe(fn(*args, **kwargs)))
    except Exception as e:  # noqa: BLE001 -- the exception is the record
        result = ("raise", type(e).__name__, str(e))
    return {"calls": tuple(rec.calls[start:]), "result": result}


# ------------------------------------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------------------------------------
R, C, G, BLOCK = 8, 64, 16, (4, 32)
_gen = torch.Generator().manual_seed(0)


def _randn(*shape, dtype=torch.float32):
    return torch.randn(*shape, generator=_gen).to(dtype)


def qargs(strategy, kind="int4", group_size=None, block=None, symmetric=True, scale_dtype=None):
    bits, typ = {"int4": (4, "int"), "int8": (8, "int"), "fp8": (8, "float"), "fp4": (4, "float"), "int3": (3, "int"),
                 "fp6": (6, "float"), "int16": (16, "int")}[kind]
    if strategy in ("group", "tensor_group") and group_size is None:
        group_size = G
    if strategy == "block" and block is None:
        block = list(BLOCK)
    return SimpleNamespace(strategy=strategy, group_size=group_size, block_structure=block, num_bits=bits, type=typ,
                           symmetric=symmetric, scale_dtype=scale_dtype, zp_dtype=None)


def scale_shape(strategy, shape, group_size=G):
    rows = math.prod(shape[:-1]) if len(shape) > 1 else 1
    cols = shape[-1]
    if strategy == "tensor":
        return (1,)
    if strategy in ("channel", "token"):
        return tuple(shape[:-1]) + (1,) if len(shape) > 1 else (1,)
    if strategy in ("group", "tensor_group"):
        return tuple(shape[:-1]) + (math.ceil(cols / group_size),) if len(shape) > 1 else (math.ceil(cols / group_size),)
    return (math.ceil(rows / BLOCK[0]), math.ceil(cols / BLOCK[1]))


def _zp(kind, shape):
    if kind == "none":
        return None
    z = torch.randint(-4, 4, shape, generator=_gen, dtype=torch.int8)
    return z if kind == "int8" else z.to(F8)


def _gs(kind):
    return {"none": None, "f32_1": torch.tensor([0.75]), "f32_0d": torch.tensor(0.75), "bf16_1": torch.tensor([0.75], dtype=torch.bfloat16),
            "f32_2": torch.tensor([0.75, 0.5])}[kind]


def _g_idx(kind, cols, group_size=G):
    if kind == "none":
        return None
    g = torch.arange(cols, dtype=torch.int64) // group_size
    return g.flip(0) if kind == "ordered" else torch.full((cols,), -1, dtype=torch.int64)


STRATEGIES = ("tensor", "channel", "group", "tensor_group", "block", "token")
ZPS = ("none", "int8", "fp8")
GSS = ("none", "f32_1", "f32_0d", "bf16_1", "f32_2")


def _scale(strategy, shape, dtype):
    return (_randn(*scale_shape(strategy, shape)).abs() + 0.05).to(dtype)


# ------------------------------------------------------------------------------------------------------------------------------
# cases
# ------------------------------------------------------------------------------------------------------------------------------
def per_tensor_cases():
    """(name, fn, args, kwargs) of every descriptor-taking per-tensor function over the grid"""
    cases = []

    def add(name, fn, *a, **k):
        cases.append((name, fn, a, k))

    # the full grid on a 2-D input: strategy x dtype x zero point x global scale
    for strategy in STRATEGIES:
        for dt in FLOATS:
            x = _randn(R, C, dtype=dt)
            sc = _scale(strategy, (R, C), dt)
            for zk in ZPS:
                zp = _zp(zk, sc.shape)
                for gk in GSS:
                    gs = _gs(gk)
                    tag = f"{strategy}/{dt}/zp={zk}/gs={gk}"
                    for kind in ("int4", "int8", "fp8"):
                        a = qargs(strategy, kind)
                        qdt = F8 if kind == "fp8" else torch.int8
                        add(f"quantize/{tag}/{kind}", ops.quantize, x, sc, zp, a, dtype=qdt, global_scale=gs)
                        add(f"fake_quantize/{tag}/{kind}", ops.fake_quantize, x, sc, zp, a, global_scale=gs)
                    add(f"quantize/{tag}/int8/dtype=None", ops.quantize, x, sc, zp, qargs(strategy, "int8"), global_scale=gs)
                    add(f"quantize_pack/{tag}/int4", ops.quantize_pack, x, sc, zp, qargs(strategy, "int4"), global_scale=gs)
                    add(f"quantize_pack_fp4/{tag}", ops.quantize_pack_fp4, x, sc, zp, qargs(strategy, "fp4"), global_scale=gs)
                    q = torch.randint(-8, 8, (R, C), generator=_gen, dtype=torch.int8)
                    add(f"dequantize/{tag}/args", ops.dequantize, q, sc, zp, qargs(strategy, "int8"), global_scale=gs)
                    add(f"dequantize/{tag}/fp8codes", ops.dequantize, q.to(F8), sc, zp, qargs(strategy, "fp8"), dtype=torch.float32,
                        global_scale=gs)
                add(f"dequantize/{strategy}/{dt}/zp={zk}/inferred", ops.dequantize, torch.randint(-8, 8, (R, C), generator=_gen, dtype=torch.int8),
                    sc, zp)

    # shapes: 1-D, 3-D, meta and empty inputs
    for strategy in STRATEGIES:
        for shape in ((C,), (2, R, C), (R, C), (0, C)):
            for device in ("cpu", "meta"):
                x = _randn(*shape, dtype=torch.bfloat16).to(device)
                sc = _scale(strategy, shape, torch.bfloat16).to(device)
                zp = _zp("int8", sc.shape).to(device)
                tag = f"{strategy}/{shape}/{device}"
                add(f"quantize/{tag}", ops.quantize, x, sc, zp, qargs(strategy, "int8"), dtype=torch.int8)
                add(f"fake_quantize/{tag}", ops.fake_quantize, x, sc, zp, qargs(strategy, "int4"))
                add(f"quantize_pack/{tag}", ops.quantize_pack, x, sc, zp, qargs(strategy, "int4"))
                add(f"quantize_pack_fp4/{tag}", ops.quantize_pack_fp4, x, sc, None, qargs(strategy, "fp4"), global_scale=_gs("f32_1"))
                q = torch.zeros(shape, dtype=torch.int8, device=device)
                add(f"dequantize/{tag}", ops.dequantize, q, sc, zp, qargs(strategy, "int8"), dtype=torch.float16)

    # g_idx with and without -1, on the group strategies
    for strategy in ("group", "tensor_group", "channel"):
        for gk in ("none", "ordered", "minus1"):
            x = _randn(R, C, dtype=torch.bfloat16)
            sc = _scale(strategy, (R, C), torch.bfloat16)
            zp = _zp("int8", sc.shape)
            gi = _g_idx(gk, C)
            tag = f"{strategy}/g_idx={gk}"
            add(f"quantize/{tag}", ops.quantize, x, sc, zp, qargs(strategy, "int4"), dtype=torch.int8, g_idx=gi)
            add(f"fake_quantize/{tag}", ops.fake_quantize, x, sc, zp, qargs(strategy, "int4"), g_idx=gi)
            add(f"quantize_pack/{tag}", ops.quantize_pack, x, sc, zp, qargs(strategy, "int4"), g_idx=gi)
            add(f"quantize_pack_fp4/{tag}", ops.quantize_pack_fp4, x, sc, None, qargs(strategy, "fp4"), g_idx=gi)
            q = torch.randint(-8, 8, (R, C), generator=_gen, dtype=torch.int8)
            add(f"dequantize/{tag}", ops.dequantize, q, sc, zp, qargs(strategy, "int4"), g_idx=gi)
            packed = torch.zeros((R, C * 4 // 32), dtype=torch.int32)
            add(f"unpack_dequantize/{tag}", ops.unpack_dequantize, packed, sc, zp, 4, (R, C), g_idx=gi)

    # error inputs: dtypes, bits, output dtypes, ragged groups, scale shapes that do not broadcast
    x = _randn(R, C, dtype=torch.bfloat16)
    sc = _scale("group", (R, C), torch.bfloat16)
    for dt in (torch.float64, torch.int8, torch.int32):
        add(f"quantize/x={dt}", ops.quantize, x.to(dt), sc, None, qargs("group"), dtype=torch.int8)
        add(f"quantize/scale={dt}", ops.quantize, x, sc.to(dt), None, qargs("group"), dtype=torch.int8)
        add(f"fake_quantize/x={dt}", ops.fake_quantize, x.to(dt), sc, None, qargs("group"))
        add(f"fake_quantize/scale={dt}", ops.fake_quantize, x, sc.to(dt), None, qargs("group"))
        add(f"quantize_pack/x={dt}", ops.quantize_pack, x.to(dt), sc, None, qargs("group"))
        add(f"quantize_pack/scale={dt}", ops.quantize_pack, x, sc.to(dt), None, qargs("group"))
        add(f"quantize_pack_fp4/x={dt}", ops.quantize_pack_fp4, x.to(dt), sc, None, qargs("group", "fp4"))
        add(f"quantize_pack_fp4/scale={dt}", ops.quantize_pack_fp4, x, sc.to(dt), None, qargs("group", "fp4"))
        add(f"dequantize/scale={dt}", ops.dequantize, torch.zeros(R, C, dtype=torch.int8), sc.to(dt), None, qargs("group"))
        add(f"dequantize/dtype={dt}", ops.dequantize, torch.zeros(R, C, dtype=torch.int8), sc, None, qargs("group"), dtype=dt)
        add(f"dequantize/codes={dt}", ops.dequantize, torch.zeros(R, C, dtype=torch.int16), sc, None, qargs("group"), dtype=dt)
        add(f"unpack_dequantize/scale={dt}", ops.unpack_dequantize, torch.zeros((R, 8), dtype=torch.int32), sc.to(dt), None, 4, (R, C))
    for kind in ("int3", "fp6", "int16", "fp8", "fp4"):
        add(f"quantize/kind={kind}", ops.quantize, x, sc, None, qargs("group", kind), dtype=torch.int8)
        add(f"quantize_pack/kind={kind}", ops.quantize_pack, x, sc, None, qargs("group", kind))
        add(f"quantize_pack_fp4/kind={kind}", ops.quantize_pack_fp4, x, sc, None, qargs("group", kind))
    add("quantize/dtype=int16", ops.quantize, x, sc, None, qargs("group"), dtype=torch.int16)
    add("quantize/ragged_group", ops.quantize, _randn(R, 40, dtype=torch.bfloat16), _scale("group", (R, 48), torch.bfloat16), None,
        qargs("group"), dtype=torch.int8)
    add("quantize/small_group", ops.quantize, _randn(R, 8, dtype=torch.bfloat16), _scale("group", (R, 8), torch.bfloat16), None,
        qargs("group"), dtype=torch.int8)
    add("quantize/bad_group_scale", ops.quantize, x, torch.ones(R, 3, dtype=torch.bfloat16), None, qargs("group"), dtype=torch.int8)
    add("quantize/bad_channel_scale", ops.quantize, x, torch.ones(R, 3, dtype=torch.bfloat16), None, qargs("channel"), dtype=torch.int8)
    add("quantize/bad_rows", ops.quantize, x, torch.ones(3, 1, dtype=torch.bfloat16), None, qargs("channel"), dtype=torch.int8)
    add("quantize/bad_block_scale", ops.quantize, x, torch.ones(3, 3, dtype=torch.bfloat16), None, qargs("block"), dtype=torch.int8)
    add("quantize/block_no_structure", ops.quantize, x, torch.ones(2, 2, dtype=torch.bfloat16), None,
        SimpleNamespace(strategy="block", group_size=None, block_structure=None, num_bits=8, type="int"), dtype=torch.int8)
    add("quantize/block_1d", ops.quantize, _randn(C, dtype=torch.bfloat16), torch.ones(1, 2, dtype=torch.bfloat16), None,
        qargs("block"), dtype=torch.int8)
    add("quantize/zp_broadcast", ops.quantize, x, _scale("channel", (R, C), torch.bfloat16), torch.zeros(1, dtype=torch.int8),
        qargs("channel"), dtype=torch.int8)
    add("fake_quantize/odd_fp4", ops.quantize_pack_fp4, _randn(R, 33, dtype=torch.bfloat16), torch.ones(R, 3, dtype=torch.bfloat16), None,
        qargs("group", "fp4"))
    add("quantize_pack_fp4/1d", ops.quantize_pack_fp4, _randn(C, dtype=torch.bfloat16), torch.ones(4, dtype=torch.bfloat16), None,
        qargs("group", "fp4"))
    add("dequantize/scale_3d", ops.dequantize, torch.zeros(R, C, dtype=torch.int8), torch.ones(2, 2, 2))
    for shape_scale in ((1, 4), (R, 4), (2, 2), (R, 1), (1,), ()):
        add(f"dequantize/infer/{shape_scale}", ops.dequantize, torch.zeros(R, C, dtype=torch.int8), torch.ones(shape_scale, dtype=torch.float16),
            dtype=torch.bfloat16)

    # unpack_dequantize: widths, over-wide and short packed words, bits, 3-D, scales of every inferred strategy
    for bits in (2, 4, 8):
        words = -(-C * bits // 32)
        for wk, w in (("exact", words), ("wide", words + 2), ("short", words - 1)):
            for ss in ((R, C // G), (R, 1), (1,), (2, 2), (1, C // G)):
                for zk in ("none", "int8"):
                    sc = torch.ones(ss, dtype=torch.float16)
                    zp = _zp(zk, sc.shape)
                    for dt in (None, torch.float32):
                        add(f"unpack_dequantize/{bits}/{wk}/{ss}/zp={zk}/dtype={dt}", ops.unpack_dequantize,
                            torch.zeros((R, w), dtype=torch.int32), sc, zp, bits, (R, C), dtype=dt)
    for device in ("cpu", "meta"):
        add(f"unpack_dequantize/3d/{device}", ops.unpack_dequantize, torch.zeros((2, R, 8), dtype=torch.int32, device=device),
            torch.ones((2, R, 4), dtype=torch.bfloat16, device=device), None, 4, (2, R, C))
        add(f"unpack_dequantize/meta/{device}", ops.unpack_dequantize, torch.zeros((R, 8), dtype=torch.int32, device=device),
            torch.ones((R, 4), dtype=torch.bfloat16, device=device), None, 4, (R, C))
    add("unpack_dequantize/int8_words", ops.unpack_dequantize, torch.zeros((R, 8), dtype=torch.int8), torch.ones(R, 4), None, 4, (R, C))
    add("unpack_dequantize/bits9", ops.unpack_dequantize, torch.zeros((R, 18), dtype=torch.int32), torch.ones(R, 4), None, 9, (R, C))
    add("unpack_dequantize/scale_int", ops.unpack_dequantize, torch.zeros((R, 8), dtype=torch.int32), torch.ones(R, 4, dtype=torch.int8),
        None, 4, (R, C))

    # FP4: stored scales, global scales, output dtypes
    for dt in FLOATS + (torch.int8,):
        for stored, sc in ((None, torch.ones(R, C // 16, dtype=torch.bfloat16)), (None, torch.ones(R, C // 16)),
                           ("fp8", torch.ones(R, C // 16).to(F8)), ("e8m0", torch.full((R, C // 32), 127, dtype=torch.uint8)),
                           ("fp8", torch.ones(R, C // 16)), ("e8m0", torch.ones(R, C // 32)), ("bogus", torch.ones(R, C // 16)),
                           (None, torch.ones(1, dtype=torch.float16)), (None, torch.ones(R, 1, dtype=torch.float16))):
            for gk in GSS:
                add(f"unpack_dequantize_fp4/{dt}/{stored}/{tuple(sc.shape)}/{sc.dtype}/gs={gk}", ops.unpack_dequantize_fp4,
                    torch.zeros((R, C // 2), dtype=torch.uint8), sc, _gs(gk), dtype=dt, stored_scale=stored)
    add("unpack_dequantize_fp4/meta", ops.unpack_dequantize_fp4, torch.zeros((R, C // 2), dtype=torch.uint8, device="meta"),
        torch.ones(R, C // 16, device="meta").to(F8), _gs("f32_1"), stored_scale="fp8")
    add("unpack_dequantize_fp4/int8", ops.unpack_dequantize_fp4, torch.zeros((R, C // 2), dtype=torch.int8), torch.ones(R, 4))
    add("unpack_dequantize_fp4/3d", ops.unpack_dequantize_fp4, torch.zeros((2, R, C // 2), dtype=torch.uint8), torch.ones(R, 4))

    # FP8 block dequantization
    for sdt in (torch.float32, torch.bfloat16):
        for dt in FLOATS + (torch.int8,):
            for rows, cols, block in ((R, C, (4, 32)), (10, 70, (4, 32)), (R, C, (8, 64))):
                for device in ("cpu", "meta"):
                    w = torch.zeros(rows, cols).to(F8).to(device)
                    si = torch.ones(math.ceil(rows / block[0]), math.ceil(cols / block[1]), dtype=sdt, device=device)
                    add(f"dequantize_block_fp8/{sdt}/{dt}/{rows}x{cols}/{block}/{device}", ops.dequantize_block_fp8, w, si, block, dtype=dt)
    add("dequantize_block_fp8/empty", ops.dequantize_block_fp8, torch.zeros(0, C).to(F8), torch.ones(0, 2), (4, 32))
    add("dequantize_block_fp8/bf16", ops.dequantize_block_fp8, torch.zeros(R, C, dtype=torch.bfloat16), torch.ones(2, 2), (4, 32))
    add("dequantize_block_fp8/bad_scale", ops.dequantize_block_fp8, torch.zeros(R, C).to(F8), torch.ones(3, 3), (4, 32))

    # the fused 2:4 + int4 pair
    for strategy in ("channel", "group", "tensor"):
        for dt in FLOATS:
            for zk in ("none", "int8"):
                x = _randn(R, C, dtype=dt)
                sc = _scale(strategy, (R, C), dt)
                zp = _zp(zk, sc.shape)
                add(f"sparse24_quantize_pack/{strategy}/{dt}/{zk}", ops.sparse24_quantize_pack, x, sc, zp, qargs(strategy, "int4"))
                sc2 = _scale(strategy, (R, C // 2) if strategy == "group" else (R, C), dt)
                zp2 = _zp(zk, sc2.shape)
                for odt in (None, torch.float32):
                    add(f"sparse24_unpack_dequantize/{strategy}/{dt}/{zk}/{odt}", ops.sparse24_unpack_dequantize,
                        torch.zeros((R, C // 16), dtype=torch.int32), torch.zeros((R, C // 8), dtype=torch.uint8), sc2, zp2, 4, (R, C), dtype=odt)
    add("sparse24_quantize_pack/fp8", ops.sparse24_quantize_pack, _randn(R, C), torch.ones(R, 1), None, qargs("channel", "fp8"))
    add("sparse24_quantize_pack/x_int", ops.sparse24_quantize_pack, torch.zeros(R, C, dtype=torch.int8), torch.ones(R, 1), None,
        qargs("channel", "int4"))
    add("sparse24_quantize_pack/cols", ops.sparse24_quantize_pack, _randn(R, 30), torch.ones(R, 1), None, qargs("channel", "int4"))
    add("sparse24_unpack_dequantize/int8", ops.sparse24_unpack_dequantize, torch.zeros((R, 4), dtype=torch.int8),
        torch.zeros((R, 8), dtype=torch.uint8), torch.ones(R, 1), None, 4, (R, C))
    return cases


def observer_cases():
    """the observers run calculate_qparams on their unfused paths, which needs resolved QuantizationArgs"""
    from compressed_tensors_b200.quantization import QuantizationArgs

    cases = []

    def add(name, fn, x, a, **k):
        try:
            a = QuantizationArgs(**{f: v for f, v in vars(a).items() if v is not None and f != "zp_dtype"})
        except Exception:  # noqa: BLE001 -- a scheme the args model refuses: keep the plain namespace
            pass
        cases.append((name, fn, (x, a), k))

    for dt in FLOATS:
        for rows, cols in ((R, C), (R, 40), (3, 24)):
            x = _randn(rows, cols, dtype=dt)
            for strategy in ("channel", "tensor", "group", "block", "token"):
                for kind in ("int4", "int8", "fp8"):
                    for sym in (True, False):
                        a = qargs(strategy, kind, group_size=8 if cols == 24 else None, symmetric=sym)
                        for pack in (False, True):
                            add(f"observe_quantize/{dt}/{rows}x{cols}/{strategy}/{kind}/sym={sym}/pack={pack}", ops.observe_quantize,
                                x, a, pack=pack)
                        if strategy in ("group", "channel", "tensor"):
                            add(f"observe_quantize_pack/{dt}/{rows}x{cols}/{strategy}/{kind}/sym={sym}", ops.observe_quantize_pack, x, a)
            for gk in ("given", "none"):
                gs = torch.tensor([0.5]) if gk == "given" else None
                add(f"observe_quantize_pack_nvfp4/{dt}/{rows}x{cols}/{gk}", ops.observe_quantize_pack_nvfp4, x,
                    qargs("tensor_group", "fp4"), global_scale=gs)
            for kind in ("fp4", "fp8"):
                add(f"observe_quantize_mx/{dt}/{rows}x{cols}/{kind}", ops.observe_quantize_mx, x,
                    qargs("group", kind, group_size=32, scale_dtype=torch.uint8))
            for kind in ("int8", "fp8", "fp4"):
                for sym in (True, False):
                    add(f"observe_tensor_qparams/{dt}/{rows}x{cols}/{kind}/{sym}", ops.observe_tensor_qparams, x, qargs("tensor", kind, symmetric=sym))
            add(f"observe_tensor_gparam/{dt}/{rows}x{cols}", lambda x, a: ops.observe_tensor_gparam(x), x, None)
            for strategy in ("token", "tensor", "group", "tensor_group"):
                add(f"dynamic_fake_quantize/{dt}/{rows}x{cols}/{strategy}", ops.dynamic_fake_quantize, x, qargs(strategy, "int8"))
    for group in (16, 32, 64, 128, 256):
        for dt in (torch.bfloat16, torch.float16):
            x = _randn(4, 256, dtype=dt)
            for sym in (True, False):
                for kind in ("int4", "int8"):
                    add(f"observe_quantize_pack/{dt}/g{group}/{kind}/{sym}", ops.observe_quantize_pack, x, qargs("group", kind, group_size=group, symmetric=sym))
    x = _randn(R, C, dtype=torch.bfloat16)
    add("observe_tensor_gparam/meta", lambda x, a: ops.observe_tensor_gparam(x), x.to("meta"), None)
    add("observe_quantize/3d", ops.observe_quantize, _randn(2, R, C), qargs("channel", "int8"))
    add("observe_quantize/fp8_pack", ops.observe_quantize, x, qargs("channel", "fp8"), pack=True)
    add("observe_quantize/attn_head", ops.observe_quantize, x, qargs("attn_head", "int8"))
    add("observe_quantize_pack/3d", ops.observe_quantize_pack, _randn(2, R, C), qargs("group", "int4"))
    add("observe_quantize_pack/token", ops.observe_quantize_pack, x, qargs("token", "int4"))
    add("observe_quantize_pack_nvfp4/args", ops.observe_quantize_pack_nvfp4, x, qargs("group", "fp4"))
    add("observe_quantize_mx/args", ops.observe_quantize_mx, x, qargs("group", "fp4", group_size=32))
    add("observe_quantize_mx/asym", ops.observe_quantize_mx, x, qargs("group", "fp4", group_size=32, scale_dtype=torch.uint8, symmetric=False))
    add("observe_quantize_mx/meta", ops.observe_quantize_mx, x.to("meta"), qargs("group", "fp8", group_size=32, scale_dtype=torch.uint8))
    add("observe_quantize/block_meta", ops.observe_quantize, x.to("meta"), qargs("block", "fp8"))
    return cases


def recipe_cases():
    """the observer descriptors that tests and tools build by name"""
    out = {}
    for dt in FLOATS:
        for shape in ((R, C), (C,), (2, R, C)):
            x = _randn(*shape, dtype=dt)
            for qt, bits in ((N.Q_INT, 8), (N.Q_FLOAT, 8), (N.Q_FP4, 4)):
                for q_dt in (None, torch.int8, F8, torch.int32):
                    for asym in (False, True):
                        out[f"_tensor_desc/{dt}/{shape}/{qt}/{q_dt}/{asym}"] = _desc(ops._tensor_desc(x, qt, bits, q_dt=q_dt, asym=asym))
        for rows, cols, bh, bw in ((256, 256, 128, 128), (300, 200, 128, 128), (16, 128, 16, 128)):
            out[f"_block_desc/{dt}/{rows}x{cols}/{bh}x{bw}"] = _desc(ops._block_desc(rows, cols, bh, bw, dt))
        for bits in (4, 8):
            out[f"_mx_desc/{dt}/{bits}"] = _desc(ops._mx_desc(257, 96, bits, dt))
    return out


# ------------------------------------------------------------------------------------------------------------------------------
# whole-model launches on host-resident modules
# ------------------------------------------------------------------------------------------------------------------------------
def _module(fmt, args, tensors: dict):
    from compressed_tensors_b200.quantization import QuantizationScheme, QuantizationStatus

    m = torch.nn.Linear(1, 1, bias=False)
    del m.weight
    for k, v in tensors.items():
        if v is not None:
            m.register_parameter(k, torch.nn.Parameter(v, requires_grad=False))
    m.quantization_scheme = QuantizationScheme(targets=["Linear"], weights=args, format=fmt)
    m.quantization_status = QuantizationStatus.FROZEN
    return m


def _state(m) -> tuple:
    from compressed_tensors_b200.utils.module import get_direct_state_dict

    return tuple(sorted((k, _describe(v)) for k, v in get_direct_state_dict(m).items()))


def model_groups():
    """(name, "compress" / "decompress", [module factories]) -- a factory so that every replay starts from fresh modules"""
    from compressed_tensors_b200.quantization import QuantizationArgs

    def qa(**k):
        return QuantizationArgs(**k)

    def w(rows, cols, dt=torch.bfloat16):
        return _randn(rows, cols, dtype=dt)

    def sc(shape, dt=torch.bfloat16):
        return (_randn(*shape).abs() + 0.05).to(dt)

    groups = []
    # pack-quantized: group / channel / tensor, symmetric and not, three dtypes
    pack = []
    for dt in FLOATS:
        for strategy, sshape, extra in (("group", (R, C // G), {"group_size": G}), ("channel", (R, 1), {}), ("tensor", (1,), {})):
            for sym in (True, False):
                a = qa(num_bits=4, type="int", symmetric=sym, strategy=strategy, **extra)
                zp = torch.randint(-4, 4, sshape, generator=_gen, dtype=torch.int8)
                pack.append((a, {"weight": w(R, C, dt), "weight_scale": sc(sshape, dt), "weight_zero_point": zp}))
    groups.append(("pack", "compress", "pack-quantized", pack))
    naive = []
    for dt in FLOATS:
        for strategy, sshape, extra in (("tensor", (1,), {}), ("channel", (R, 1), {}), ("block", (2, 2), {"block_structure": [4, 32]}),
                                        ("group", (R, C // G), {"group_size": G})):
            for typ, bits, sym in (("float", 8, True), ("int", 8, True), ("int", 8, False)):
                a = qa(num_bits=bits, type=typ, symmetric=sym, strategy=strategy, **extra)
                zp = torch.zeros(sshape, dtype=F8 if typ == "float" else torch.int8)
                naive.append((a, {"weight": w(R, C, dt), "weight_scale": sc(sshape, dt), "weight_zero_point": zp}))
    groups.append(("naive", "compress", "naive-quantized", naive))
    groups.append(("float", "compress", "float-quantized", naive[:6]))
    nv = []
    for dt in FLOATS:
        for gs in (torch.tensor([0.5]), None):
            a = qa(num_bits=4, type="float", symmetric=True, strategy="tensor_group", group_size=16)
            nv.append((a, {"weight": w(R, C, dt), "weight_scale": sc((R, C // 16), dt), "weight_global_scale": gs}))
    groups.append(("nvfp4", "compress", "nvfp4-pack-quantized", nv))
    mx = []
    for dt in FLOATS:
        a = qa(num_bits=4, type="float", symmetric=True, strategy="group", group_size=32, scale_dtype=torch.uint8)
        mx.append((a, {"weight": w(R, C, dt), "weight_scale": torch.full((R, C // 32), 0.25, dtype=dt)}))
    groups.append(("mxfp4", "compress", "mxfp4-pack-quantized", mx))

    # decompression, from hand-made compressed tensors
    dpack = []
    for dt in FLOATS:
        for strategy, sshape, extra in (("group", (R, C // G), {"group_size": G}), ("channel", (R, 1), {}), ("tensor", (1,), {})):
            for sym in (True, False):
                for bits in (4, 8):
                    a = qa(num_bits=bits, type="int", symmetric=sym, strategy=strategy, **extra)
                    t = {"weight_packed": torch.randint(-2**31, 2**31 - 1, (R, C * bits // 32), generator=_gen, dtype=torch.int32),
                         "weight_shape": torch.tensor([R, C]), "weight_scale": sc(sshape, dt)}
                    if not sym:
                        zrows = sshape[0] if strategy == "tensor" else -(-sshape[0] * bits // 32)
                        t["weight_zero_point"] = torch.zeros((zrows, sshape[1]) if len(sshape) == 2 else sshape, dtype=torch.int32) \
                            if strategy != "tensor" else torch.zeros(sshape, dtype=torch.int8)
                    dpack.append((a, t))
    groups.append(("dpack", "decompress", "pack-quantized", dpack))
    dnaive = []
    for dt in FLOATS:
        for strategy, sshape, extra in (("tensor", (1,), {}), ("channel", (R, 1), {}), ("block", (2, 2), {"block_structure": [4, 32]}),
                                        ("group", (R, C // G), {"group_size": G})):
            for typ, qdt, sym in (("float", F8, True), ("int", torch.int8, True), ("int", torch.int8, False)):
                a = qa(num_bits=8, type=typ, symmetric=sym, strategy=strategy, **extra)
                t = {"weight": torch.zeros(R, C).to(qdt), "weight_scale": sc(sshape, dt)}
                if not sym:
                    t["weight_zero_point"] = torch.zeros(sshape, dtype=torch.int8)
                dnaive.append((a, t))
    groups.append(("dnaive", "decompress", "naive-quantized", dnaive))
    dnv = []
    for gs in (torch.tensor([0.5]), None, torch.tensor(0.5)):
        for sdt in (F8, torch.bfloat16):
            a = qa(num_bits=4, type="float", symmetric=True, strategy="tensor_group", group_size=16)
            dnv.append((a, {"weight_packed": torch.zeros((R, C // 2), dtype=torch.uint8), "weight_scale": torch.ones(R, C // 16).to(sdt),
                            "weight_global_scale": gs}))
    groups.append(("dnvfp4", "decompress", "nvfp4-pack-quantized", dnv))
    dmx = [(qa(num_bits=4, type="float", symmetric=True, strategy="group", group_size=32, scale_dtype=torch.uint8),
            {"weight_packed": torch.zeros((R, C // 2), dtype=torch.uint8), "weight_scale": torch.full((R, C // 32), 127, dtype=torch.uint8)})]
    groups.append(("dmxfp4", "decompress", "mxfp4-pack-quantized", dmx))

    # inputs on which the whole-model path and the per-module path disagreed
    groups.append(("pack_f64_weight", "compress", "pack-quantized",
                   [(qa(num_bits=4, type="int", symmetric=True, strategy="group", group_size=G),
                     {"weight": w(R, C, torch.float64), "weight_scale": sc((R, C // G))})]))
    groups.append(("pack_f64_scale", "compress", "pack-quantized",
                   [(qa(num_bits=4, type="int", symmetric=True, strategy="group", group_size=G),
                     {"weight": w(R, C), "weight_scale": sc((R, C // G), torch.float64)})]))
    groups.append(("naive_f64_weight", "compress", "naive-quantized",
                   [(qa(num_bits=8, type="int", symmetric=True, strategy="channel"),
                     {"weight": w(R, C, torch.float64), "weight_scale": sc((R, 1))})]))
    groups.append(("pack_int_scale", "compress", "pack-quantized",
                   [(qa(num_bits=4, type="int", symmetric=True, strategy="group", group_size=G),
                     {"weight": w(R, C), "weight_scale": torch.ones((R, C // G), dtype=torch.int8)})]))
    groups.append(("naive_int_weight", "compress", "naive-quantized",
                   [(qa(num_bits=8, type="int", symmetric=True, strategy="channel"),
                     {"weight": torch.ones(R, C, dtype=torch.int8), "weight_scale": sc((R, 1))})]))
    groups.append(("nvfp4_int_scale", "compress", "nvfp4-pack-quantized",
                   [(qa(num_bits=4, type="float", symmetric=True, strategy="tensor_group", group_size=16),
                     {"weight": w(R, C), "weight_scale": torch.ones((R, C // 16), dtype=torch.int8), "weight_global_scale": torch.tensor([0.5])})]))
    groups.append(("pack_float_args", "compress", "pack-quantized",
                   [(qa(num_bits=8, type="float", symmetric=True, strategy="channel"), {"weight": w(R, C), "weight_scale": sc((R, 1))})]))
    groups.append(("nvfp4_f64_weight", "compress", "nvfp4-pack-quantized",
                   [(qa(num_bits=4, type="float", symmetric=True, strategy="tensor_group", group_size=16),
                     {"weight": w(R, C, torch.float64), "weight_scale": sc((R, C // 16)), "weight_global_scale": torch.tensor([0.5])})]))
    groups.append(("dpack_wide_words", "decompress", "pack-quantized",
                   [(qa(num_bits=4, type="int", symmetric=True, strategy="group", group_size=G),
                     {"weight_packed": torch.zeros((R, C * 4 // 32 + 2), dtype=torch.int32), "weight_shape": torch.tensor([R, C]),
                      "weight_scale": sc((R, C // G))})]))
    groups.append(("dpack_int_scale", "decompress", "pack-quantized",
                   [(qa(num_bits=4, type="int", symmetric=True, strategy="group", group_size=G),
                     {"weight_packed": torch.zeros((R, C * 4 // 32), dtype=torch.int32), "weight_shape": torch.tensor([R, C]),
                      "weight_scale": torch.ones((R, C // G), dtype=torch.int8)})]))
    groups.append(("dpack_float_words", "decompress", "pack-quantized",
                   [(qa(num_bits=4, type="int", symmetric=True, strategy="group", group_size=G),
                     {"weight_packed": torch.zeros((R, C * 4 // 32)), "weight_shape": torch.tensor([R, C]),
                      "weight_scale": sc((R, C // G))})]))
    groups.append(("dnvfp4_uint8_scale", "decompress", "nvfp4-pack-quantized",
                   [(qa(num_bits=4, type="float", symmetric=True, strategy="tensor_group", group_size=16),
                     {"weight_packed": torch.zeros((R, C // 2), dtype=torch.uint8), "weight_scale": torch.full((R, C // 16), 127, dtype=torch.uint8),
                      "weight_global_scale": torch.tensor([0.5])})]))
    groups.append(("dmxfp4_fp8_scale", "decompress", "mxfp4-pack-quantized",
                   [(qa(num_bits=4, type="float", symmetric=True, strategy="group", group_size=32, scale_dtype=torch.uint8),
                     {"weight_packed": torch.zeros((R, C // 2), dtype=torch.uint8), "weight_scale": torch.ones(R, C // 32).to(F8)})]))
    groups.append(("dnaive_int_scale", "decompress", "naive-quantized",
                   [(qa(num_bits=8, type="int", symmetric=True, strategy="channel"),
                     {"weight": torch.zeros(R, C, dtype=torch.int8), "weight_scale": torch.ones((R, 1), dtype=torch.int32)})]))
    return groups


def run_model_group(rec, direction, fmt, specs) -> dict:
    from compressed_tensors_b200.compressors.model_compressors.batched import compress_modules_batched, decompress_modules_batched
    from compressed_tensors_b200.config import CompressionFormat

    mods = [_module(CompressionFormat(fmt), a, {k: v.clone() if v is not None else None for k, v in t.items()}) for a, t in specs]
    fn = compress_modules_batched if direction == "compress" else decompress_modules_batched
    r = run(rec, fn, mods)
    r["modules"] = tuple(_state(m) for m in mods)
    return r


def collect() -> dict:
    """every record, by case name"""
    global _gen
    _gen = torch.Generator().manual_seed(0)
    records = {}
    with recording() as rec:
        for name, fn, a, k in per_tensor_cases() + observer_cases():
            assert name not in records, name
            records[name] = run(rec, fn, *a, **k)
        for name, d in recipe_cases().items():
            records[name] = {"calls": (), "result": ("desc", d)}
    for name, direction, fmt, specs in model_groups():
        with recording(pretend_cuda=True) as rec:
            records[f"batched/{name}"] = run_model_group(rec, direction, fmt, specs)
    return records


if __name__ == "__main__":
    from tests.golden import _gz

    recs = collect()
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "descriptors.pt.gz")
    with open(path, "wb") as f:
        f.write(_gz({"cases": recs}))
    print(f"{len(recs)} records -> {path}")
