#!/usr/bin/env python
"""Launch the round-2 kernels a few times each so that ncu can capture one launch per kernel:
    ncu --set full --clock-control none --import-source on -k regex:'ring|lookback|stream_tma|minmax' -c 12 -o gpurun_out/r2_sparse python tools/profile_sparse.py
one [14336, 8192] bf16 tensor for the bitmask kernels, 4 Llama-3-8B layers for the 2:4 + int4 multi-tensor launches, one L2-sized and
one larger tensor for the per-tensor observer."""
import os
import sys
from types import SimpleNamespace

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from compressed_tensors_b200 import _native as N, ops  # noqa: E402
from compressed_tensors_b200.utils.semi_structured_conversions import mask_creator  # noqa: E402

dev = torch.device("cuda", 0)
torch.manual_seed(0)
sp = (torch.randn(14336, 8192, device=dev) * 0.02).to(torch.bfloat16)
un = torch.where(torch.rand(sp.shape, device=dev) < 0.5, sp, torch.zeros_like(sp))
vals, mask, offs = ops.bitmask_compress(un)
for _ in range(2):
    ops.bitmask_compress(un, exact=False)
    ops.bitmask_decompress(vals, mask, offs, un.shape)
torch.cuda.synchronize()

a = SimpleNamespace(strategy="group", group_size=128, block_structure=None, num_bits=4, type="int", symmetric=True)
shapes = [(4096, 4096), (1024, 4096), (1024, 4096), (4096, 4096), (14336, 4096), (14336, 4096), (4096, 14336)] * 4
c24, d24, keep = [], [], []
for i, (r, c) in enumerate(shapes):
    w = (torch.randn(r, c, device=dev) * 0.02).to(torch.bfloat16)
    w = w * mask_creator(w).to(w.dtype)
    sc = (w.unflatten(-1, (-1, 128)).abs().amax(-1).float() / 7.5).bfloat16()
    pk = torch.empty(r, c // 16, dtype=torch.int32, device=dev)
    bm = torch.empty(r, c // 8, dtype=torch.uint8, device=dev)
    bk = torch.empty_like(w)
    d1 = ops._quantize_pack_call(w, sc, None, a).desc
    # the 2:4 stream holds half the words: the recipe reads only the shape of a dense-width placeholder
    d2 = ops._unpack_dequantize_call(torch.empty((r, c // 8), dtype=torch.int32, device="meta"), sc, None, 4, (r, c)).desc
    d1.aux = d2.aux = bm.data_ptr()
    c24.append((d1, w, sc, None, pk)); d24.append((d2, pk, sc, None, bk)); keep.append(bm)
pc, pd = ops.BatchedPlan(N.OP_SPARSE24_QUANTIZE_PACK, c24, 0), ops.BatchedPlan(N.OP_SPARSE24_UNPACK_DEQUANTIZE, d24, 0)
for _ in range(2):
    pc.run(); pd.run()
torch.cuda.synchronize()

f8 = SimpleNamespace(strategy="tensor", group_size=None, block_structure=None, num_bits=8, type="float", symmetric=True)
for shape in ((4096, 4096), (14336, 8192)):
    x = (torch.randn(shape, device=dev) * 0.02).to(torch.bfloat16)
    for _ in range(2):
        ops.observe_quantize(x, f8)
torch.cuda.synchronize()
print("launched", N.launch_count())
