"""
The headline multi-tensor ops on `layers` Llama-3-8B layers (>> L2), as ops.batched problem lists:
the inputs tools/jitter.py times and tools/profile_ops.py launches.
"""
import os
import sys
from types import SimpleNamespace

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from compressed_tensors_b200 import _native as N  # noqa: E402
from compressed_tensors_b200 import ops  # noqa: E402


def build_problems(layers: int):
    dev = torch.device("cuda", 0)
    ws, scs = bench.make_weights(dev, layers, 1000)
    n = sum(w.numel() for w in ws)
    qa = bench.args_w4()
    outs = [torch.empty(w.shape[0], w.shape[1] // 8, dtype=torch.int32, device=dev) for w in ws]
    back = [torch.empty_like(w) for w in ws]
    f8 = SimpleNamespace(strategy="tensor", group_size=None, block_structure=None, num_bits=8, type="float", symmetric=True)
    s8 = [(w.abs().max().float() / 448).bfloat16().reshape(1) for w in ws]
    q8 = [torch.empty(w.shape, dtype=torch.float8_e4m3fn, device=dev) for w in ws]
    P = {"quantpack": [], "unpackdeq": [], "fp8_q": [], "fp8_dq": [], "fake_w4": [], "observe_qp": [], "nvfp4_qp": [], "nvfp4_ud": []}
    nv = SimpleNamespace(strategy="tensor_group", group_size=16, block_structure=None, num_bits=4, type="float", symmetric=True)
    keep = []
    sc_out = [torch.empty_like(s) for s in scs]
    for w, sc, o, b, s, q, so in zip(ws, scs, outs, back, s8, q8, sc_out):
        qp = ops._quantize_pack_call(w, sc, None, qa).desc
        P["observe_qp"].append((qp, w, so, None, o))      # the observer writes the scale: same descriptor, scale as an output
        P["quantpack"].append((qp, w, sc, None, o))
        P["unpackdeq"].append((ops._unpack_dequantize_call(o, sc, None, 4, w.shape).desc, o, sc, None, b))
        P["fake_w4"].append((ops._fake_quantize_call(w, sc, None, qa).desc, w, sc, None, b))
        P["fp8_q"].append((ops._quantize_call(w, s, None, f8, dtype=torch.float8_e4m3fn).desc, w, s, None, q))
        g = (448.0 * 6.0 / w.abs().max().float()).reshape(1)
        s8n = (w.unflatten(-1, (-1, 16)).abs().amax(-1).float() / 6.0 * g).clamp(2.0 ** -9, 448.0).to(torch.float8_e4m3fn)
        sbn = s8n.to(torch.bfloat16)
        nib = torch.empty(w.shape[0], w.shape[1] // 2, dtype=torch.uint8, device=dev)
        dn = ops._quantize_pack_fp4_call(w, sbn, None, nv, global_scale=g).desc
        du = ops._unpack_dequantize_fp4_call(nib, s8n, g, torch.bfloat16, stored_scale="fp8").desc
        dn.global_scale = du.global_scale = g.data_ptr()   # the recipes leave the device pointer to the launch
        keep.append(g)
        P["nvfp4_qp"].append((dn, w, sbn, None, nib))
        P.setdefault("nvfp4_observe_qp", []).append((ops._nvfp4_observe_desc(*w.shape, w.dtype, g.data_ptr()), w, torch.empty_like(s8n), None, nib))
        P["nvfp4_ud"].append((du, nib, s8n, None, b))
        P["fp8_dq"].append((ops._dequantize_call(q, s, None, f8).desc, q, s, None, b))
    OPS = {"quantpack": (N.OP_QUANTIZE_PACK, 2.515625), "unpackdeq": (N.OP_UNPACK_DEQUANTIZE, 2.515625),
           "observe_qp": (N.OP_OBSERVE_QUANTIZE_PACK, 2.515625), "fp8_q": (N.OP_QUANTIZE, 3.0), "fp8_dq": (N.OP_DEQUANTIZE, 3.0), "fake_w4": (N.OP_FAKE_QUANTIZE, 4.0 + 2 / 128),
           "nvfp4_qp": (N.OP_QUANTIZE_PACK_FP4, 2 + 2 / 16 + 0.5), "nvfp4_observe_qp": (N.OP_OBSERVE_QUANTIZE_PACK_FP4, 2 + 1 / 16 + 0.5), "nvfp4_ud": (N.OP_UNPACK_DEQUANTIZE_FP4, 0.5 + 1 / 16 + 2)}
    P["_keep"] = keep   # global-scale tensors referenced by address from the descriptors
    return P, OPS, n

