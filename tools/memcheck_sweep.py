"""One pass over every kernel family at small, deliberately ragged and at pipeline-sized shapes, meant to run under
    compute-sanitizer --tool memcheck --error-exitcode 9 python tools/memcheck_sweep.py
so that out-of-bounds / misaligned accesses of the generic kernels' tails and of the TMA ring's last tiles show up.  Results are
not checked here (the -m gpu tests do that against the oracle); the script only has to touch every code path once."""
import itertools
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from compressed_tensors_b200 import _native as N, ops  # noqa: E402
from compressed_tensors_b200.quantization import QuantizationArgs  # noqa: E402

DEV = torch.device("cuda", 0)


def qa(**kw):
    kw.setdefault("symmetric", True)
    return QuantizationArgs(**kw)


def scale_for(x, shape, qmax, dt=None):
    return ((torch.rand(shape, device=DEV) + 0.25) * float(x.float().abs().max()) / qmax).to(dt or x.dtype)


def quant_family(rows, cols, dt):
    x = torch.randn(rows, cols, device=DEV).to(dt)
    for bits, qtype, qmax, qdt in ((4, "int", 7.5, torch.int8), (8, "int", 127.5, torch.int8), (8, "float", 448.0, torch.float8_e4m3fn)):
        cases = [(qa(num_bits=bits, type=qtype, strategy="tensor"), (1,)), (qa(num_bits=bits, type=qtype, strategy="channel"), (rows, 1))]
        for g in (32, 128):
            if cols % g == 0:
                cases.append((qa(num_bits=bits, type=qtype, strategy="group", group_size=g), (rows, cols // g)))
        cases.append((qa(num_bits=bits, type=qtype, strategy="block", block_structure=[128, 128]), (-(-rows // 128), -(-cols // 128))))
        for a, shape in cases:
            s = scale_for(x, shape, qmax)
            zp = torch.randint(-4, 4, shape, device=DEV, dtype=torch.int8) if qtype == "int" and shape != (1,) else None
            for z in (None, zp):
                q = ops.quantize(x, s, z, a, dtype=qdt)
                ops.dequantize(q, s, z, args=a)
                ops.fake_quantize(x, s, z, a)
                if qtype == "int" and cols % (32 // bits) == 0:
                    p = ops.quantize_pack(x, s, z, a)
                    if a.strategy != "block" or (rows % 128 == 0 and cols % 128 == 0):  # args=None inference needs whole blocks (forward.py:118-120)
                        ops.unpack_dequantize(p, s, z, bits, (rows, cols))
    for bits in (2, 3, 4, 8):
        codes = torch.randint(-(2 ** (bits - 1)), 2 ** (bits - 1), (rows, cols), device=DEV, dtype=torch.int8)
        for dim in (0, 1):
            p = ops.pack_to_int32(codes, bits, packed_dim=dim)
            ops.unpack_from_int32(p, bits, (rows, cols), packed_dim=dim)


def fp4_family(rows, cols, dt):
    x = torch.randn(rows, cols, device=DEV).to(dt)
    ops.unpack_fp4_from_uint8(ops.pack_fp4_to_uint8(ops.cast_to_fp4(x)), rows, cols, dt)
    if cols % 16 == 0:
        a = qa(num_bits=4, type="float", strategy="tensor_group", group_size=16, scale_dtype=torch.float8_e4m3fn)
        gs = torch.tensor([448.0 * 6.0 / float(x.float().abs().max())], device=DEV)
        s8 = (x.float().reshape(rows, cols // 16, 16).abs().amax(-1) / 6.0 * gs).clamp(2 ** -9, 448).to(torch.float8_e4m3fn)
        for s in (s8.to(dt), s8.float()):
            p = ops.quantize_pack_fp4(x, s, None, a, global_scale=gs)
            ops.unpack_dequantize_fp4(p, s, gs, dtype=dt)
        ops.unpack_dequantize_fp4(p, s8, gs, stored_scale="fp8")
        ops.observe_quantize_pack_nvfp4(x, a)
    if cols % 32 == 0:
        a = qa(num_bits=4, type="float", strategy="group", group_size=32, scale_dtype=torch.uint8, zp_dtype=torch.uint8)
        e = torch.randint(118, 130, (rows, cols // 32), device=DEV, dtype=torch.uint8)
        s = ops.decompress_mx_scale(e)
        ops.compress_mx_scale(s)
        p = ops.quantize_pack_fp4(x, s.to(dt), None, a)
        ops.unpack_dequantize_fp4(p, e, None, stored_scale="e8m0")


def sparse_family(rows, cols, dt):
    x = torch.randn(rows, cols, device=DEV).to(dt)
    if cols % 4 == 0:
        v, m = ops.sparse24_compress(x)
        ops.sparse24_decompress(v, m, (rows, cols))
    u = torch.where(torch.rand(rows, cols, device=DEV) < 0.5, x, torch.zeros_like(x))
    v, m, o = ops.bitmask_compress(u)
    ops.bitmask_decompress(v, m, o, (rows, cols))
    b = torch.rand(rows, cols, device=DEV) < 0.3
    ops.unpack_bitmasks(ops.pack_bitmasks(b), (rows, cols))
    # round 2: one-pass bitmask (ring kernel + look-back), fused 2:4 + int4
    for density in (0.0, 0.07, 1.0):
        u = torch.where(torch.rand(rows, cols, device=DEV) < density, x, torch.zeros_like(x))
        v, m, o, n = ops.bitmask_compress(u, exact=False)
        ops.bitmask_decompress(v[: int(n.item())].clone(), m, o, (rows, cols))
    if cols % 4 == 0 and dt != torch.float32:
        for a, shape in ((qa(num_bits=4, type="int", strategy="channel"), (rows, 1)), (qa(num_bits=4, type="int", strategy="group", group_size=32), (rows, max(cols // 32, 1)))):
            if a.strategy == "group" and cols % 32 != 0:
                continue
            s = scale_for(x, shape, 7.5)
            z = torch.randint(-4, 4, shape, device=DEV, dtype=torch.int8)
            for zz in (None, z):
                pk, bm = ops.sparse24_quantize_pack(x, s, zz, a)
                ops.sparse24_unpack_dequantize(pk, bm, s, zz, 4, (rows, cols))


def observer_family(rows, cols, dt):
    x = torch.randn(rows, cols, device=DEV).to(dt)
    for sym in (True, False):
        for g in (32, 128):
            if cols % g == 0:
                for bits in (4, 8):
                    ops.observe_quantize_pack(x, qa(num_bits=bits, type="int", strategy="group", group_size=g, symmetric=sym))
        for kw, pack in ((dict(num_bits=8, type="int"), False), (dict(num_bits=4, type="int"), True)):
            ops.observe_quantize(x, qa(strategy="channel", symmetric=sym, **kw), pack=pack)
    ops.observe_quantize(x, qa(strategy="channel", num_bits=8, type="float"))
    # round 2: per-tensor observers (grid-wide reduction + last-CTA qparams), NVFP4 global scale on the device
    for kw, pack in ((dict(num_bits=8, type="float"), False), (dict(num_bits=8, type="int", symmetric=False), False), (dict(num_bits=4, type="int"), True)):
        ops.observe_quantize(x, qa(strategy="tensor", **kw), pack=pack)
    if (rows * cols) % 8 == 0:
        ops.observe_tensor_gparam(x)


def converter_family(rows, cols):
    w = torch.randn(rows, cols, device=DEV).to(torch.float8_e4m3fn)
    s = torch.rand(-(-rows // 128), -(-cols // 128), device=DEV) * 0.01 + 1e-4
    ops.dequantize_block_fp8(w, s, (128, 128), torch.bfloat16)
    if cols % 8 == 0:
        q = torch.randint(-2 ** 31, 2 ** 31 - 1, (rows, cols // 8), device=DEV, dtype=torch.int64).to(torch.int32)
        ops.awq_repack(q)
        ops.awq_repack_zeros(q[: max(1, rows // 128)])


def batched_family(dt):
    """the multi-tensor persistent launch (what ModelCompressor.compress_model uses) with tensors of unequal size"""
    a = qa(num_bits=4, type="int", strategy="group", group_size=128)
    probs = []
    for rows, cols in ((4096, 4096), (1024, 4096), (14336, 4096), (40, 256), (4096, 14336)):
        x = torch.randn(rows, cols, device=DEV).to(dt)
        s = scale_for(x, (rows, cols // 128), 7.5)
        out = torch.empty(rows, cols // 8, dtype=torch.int32, device=DEV)
        p = ops._resolve(x, s, None, a, None)
        probs.append((ops._desc(p, dt, dt, None, dt, torch.int8, None, N.Q_INT, 4), x, s, None, out))
    ops.batched(N.OP_QUANTIZE_PACK, probs, 0)
    # round 2: the fused 2:4 + int4 ops as multi-tensor launches (bitmask in desc.aux)
    c24, d24, keep = [], [], []
    for d, x, s, _, _ in probs:
        rows, cols = x.shape
        if cols % 32 or (rows * cols) % 64:
            continue
        pk = torch.empty(rows, cols // 16, dtype=torch.int32, device=DEV)
        bm = torch.empty(rows, cols // 8, dtype=torch.uint8, device=DEV)
        bk = torch.empty_like(x)
        p = ops._resolve(x, s, None, a, None)
        d1 = ops._desc(p, dt, dt, None, dt, torch.int8, None, N.Q_INT, 4)
        d2 = ops._desc(p, None, dt, None, None, torch.int8, dt, N.Q_INT, 4)
        d1.aux = d2.aux = bm.data_ptr()
        c24.append((d1, x, s, None, pk)); d24.append((d2, pk, s, None, bk)); keep.append(bm)
    ops.batched(N.OP_SPARSE24_QUANTIZE_PACK, c24, 0)
    ops.batched(N.OP_SPARSE24_UNPACK_DEQUANTIZE, d24, 0)


def transform_family(dt):
    """ct_hadamard_transform: every order in both precisions with one-row partial last tiles, fp64 at 2^15 on more tiles than its
    grid of 2 x SMs (CTAs reuse their global scratch slice), rows one element off alignment (element loads and stores) with sign,
    perm and inverse, and strided [B, H, S, D] views with head blocking and decode"""
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    for log2_n in range(1, 16):
        n = 1 << log2_n
        rows = 2 * sms + 7 if log2_n == 15 else (4096 // n + 1 if n < 4096 else 3)
        x = torch.randn(rows, n, device=DEV).to(dt)
        q = (torch.randint(0, 2, (n,), device=DEV) * 2 - 1).to(torch.int8)
        perm = torch.randperm(n, device=DEV)
        odd = torch.randn(3 * n + 1, device=DEV).to(dt)[1:].view(3, n) if n in (2, 16, 128, 4096) else None
        for precision in (torch.float32, torch.float64):
            for sign, p, inverse in ((None, None, False), (q, perm, False), (q, perm, True)):
                ops.hadamard_transform(x, n, sign, p, inverse, precision)
                if odd is not None:
                    ops.hadamard_transform(odd, n, sign, p, inverse, precision)
    for B, H, S, D, n in ((2, 8, 33, 64, 64), (2, 4, 17, 256, 64), (3, 8, 1, 256, 64), (1, 32, 256, 128, 128)):
        x = torch.randn(B, S, H, D, device=DEV).to(dt).transpose(1, 2)
        q = (torch.randint(0, 2, (n,), device=DEV) * 2 - 1).to(torch.int8)
        for precision in (torch.float32, torch.float64):
            ops.hadamard_transform(x, n, q, torch.randperm(n, device=DEV), True, precision)


def heads_family(dt):
    """ct_fake_quantize_heads: every zero-point kind (none, int8, all-zero float8) and rounding width, per tensor and per head, on
    K / V pairs of unequal shapes, with an empty first job, and on one tensor"""
    k = torch.randn(1, 37, 8, 128, device=DEV).to(dt).transpose(1, 2)
    v = torch.randn(2, 5, 4, 64, device=DEV).to(dt).transpose(1, 2)
    empty = torch.randn(2, 0, 4, 64, device=DEV).to(dt).transpose(1, 2)
    schemes = [(8, "int", True, None), (8, "int", False, torch.int8), (7, "int", True, None), (4, "int", False, torch.int8),
               (2, "int", True, None), (8, "float", True, None), (8, "float", True, torch.float8_e4m3fn)]
    for strategy in ("tensor", "attn_head"):
        for bits, qtype, sym, zdt in schemes:
            a = qa(num_bits=bits, type=qtype, strategy=strategy, symmetric=sym)

            def qp(x):
                shape = (x.shape[1], 1, 1) if strategy == "attn_head" else (1,)
                s = ((torch.rand(shape, device=DEV) + 0.1) / 2 ** (bits - 1)).to(dt)
                z = None if zdt is None else (torch.randint(-2, 2, shape, device=DEV, dtype=torch.int8) if zdt == torch.int8
                                              else torch.zeros(shape, device=DEV, dtype=zdt))
                return s, z
            for pair in ((k, v), (v, k), (empty, v), (k,)):
                sz = [qp(x) for x in pair]
                ops.fake_quantize_heads(list(pair), [s for s, _ in sz], [z for _, z in sz], a)


def dynamic_family(dt):
    """ct_dynamic_fake_quantize: every strategy it takes (TOKEN up to the widest 32768-column row on the 512-thread CTA, GROUP 16..128
    on every element rule, TENSOR), ragged row counts that end inside a warp span and a CTA"""
    schemes = [dict(num_bits=8, type="int", strategy="token"), dict(num_bits=8, type="int", strategy="token", symmetric=False),
               dict(num_bits=8, type="float", strategy="token"), dict(num_bits=8, type="float", strategy="group", group_size=128),
               dict(num_bits=8, type="int", strategy="group", group_size=64, symmetric=False),
               dict(num_bits=4, type="float", strategy="tensor_group", group_size=16, scale_dtype=torch.float8_e4m3fn, zp_dtype=torch.float8_e4m3fn),
               dict(num_bits=4, type="float", strategy="group", group_size=32, scale_dtype=torch.uint8, zp_dtype=torch.uint8),
               dict(num_bits=8, type="float", strategy="group", group_size=32, scale_dtype=torch.uint8, zp_dtype=torch.uint8),
               dict(num_bits=8, type="int", strategy="tensor", symmetric=False)]
    for shape, planted in itertools.product(((1, 1, 128), (3, 7, 4104), (2, 5, 1040 * 16), (1, 3, 32768), (1001, 160), (7, 3, 2, 64)),
                                            (False, True)):
        x = torch.randn(shape, device=DEV).to(dt)
        if planted:   # NaN and +-inf take the NaN-propagating reductions and clamps
            flat = x.view(-1)
            flat[::97], flat[5::131], flat[7::151] = float("nan"), float("inf"), float("-inf")
        for kw in schemes:
            a = qa(dynamic=True, **kw)
            if kw["strategy"] in ("group", "tensor_group") and shape[-1] % kw["group_size"]:
                continue
            gs = torch.full((1,), 64.0, device=DEV) if kw.get("scale_dtype") == torch.float8_e4m3fn else None
            ops.dynamic_fake_quantize(x, a, global_scale=gs)


FAILED = []


def attempt(fn, *a):
    """a Python-level rejection (unsupported combination, a bug in this script) must not hide the rest of the sweep"""
    try:
        fn(*a)
    except Exception as e:  # noqa: BLE001
        FAILED.append(f"{fn.__name__}{a}: {type(e).__name__}: {str(e)[:200]}")


def main():
    torch.cuda.set_device(0)
    torch.manual_seed(0)
    shapes = [(1, 8), (3, 40), (33, 136), (257, 1000), (64, 4096), (1024, 2048)]
    for dt in (torch.bfloat16, torch.float16, torch.float32):
        for rows, cols in shapes:
            attempt(quant_family, rows, cols, dt)
            attempt(fp4_family, rows, cols - cols % 2, dt)
            attempt(sparse_family, rows, cols, dt)
            if dt != torch.float32:
                attempt(observer_family, rows, cols, dt)
        attempt(transform_family, dt)
        attempt(heads_family, dt)
        if dt != torch.float32:
            attempt(dynamic_family, dt)
        torch.cuda.synchronize()
        print(f"{dt}: launches so far {N.launch_count()}", flush=True)
    for rows, cols in ((128, 128), (200, 384), (1024, 2048)):
        attempt(converter_family, rows, cols)
    attempt(batched_family, torch.bfloat16)
    torch.cuda.synchronize()
    for f in FAILED:
        print("PYTHON-LEVEL FAILURE", f, flush=True)
    print(f"memcheck sweep done: {N.launch_count()} library launches, {len(FAILED)} python-level failures", flush=True)


if __name__ == "__main__":
    main()
