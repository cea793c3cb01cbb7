#!/usr/bin/env python
"""
Walsh-Hadamard transforms on the H100: ops.hadamard_transform (ct_hadamard_transform) against the reference's dense formula on the same
GPU (cast to fp32 -> matmul with the n x n matrix -> divide by sqrt(n) -> cast back), on Llama-3-8B shapes.

    python tools/transform_bench.py [--iters 50] [--warmup 10] [--json out.json]

Cases: online R1 on activations [8192, 4096] bf16 (n = 4096); R3 on q / k in the transposed [B, 32 | 8, S, 128] layout the attention
hooks receive, prefill (B=1, S=8192) and decode (B=64, S=1); fp64 fusion (weight_input, n = 4096) of every 4096-input weight of the
8B model (q, k, v, o, gate, up per layer: 32 layers, one layer's tensors reused).  Orders that are not powers of two, n = K * 2^m with
a K x K +-1 core (ops.hadamard_transform(..., core=C), M = diag(Q) . (C ⊗ H_{2^m})^T; the core is a seeded +-1 matrix, which costs the
kernel what a Hadamard one does): online R4 on the down_proj input of Llama-3-8B [8192, 14336] (K = 224), Llama-3-70B [4096, 28672]
(K = 224) and Llama-2-7B [8192, 11008] (K = 172), in bf16, and the fp64 fusion (weight_input) of the 32 down_proj weights
[4096, 14336] of Llama-3-8B (one reused).  For these the compute bound is also given: K + m additions per element at the data sheet's
67 TFLOP/s FP32 (33.5 T additions / s) or 34 TFLOP/s FP64.  Per case: time per call from CUDA events after
warm-up, the algorithmic bandwidth (read + write of the tensor), its share of 3.35 TB/s and of the copy rate of tools/hbm_ceilings.py
measured in the same run, the dense formula's time, and whether both outputs lie within the parity bound of DESIGN.md section 3.  The
card, its power limit and max SM clock are printed with the numbers.
"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from compressed_tensors_b200 import ops  # noqa: E402
from compressed_tensors_b200.transform.utils.hadamard import deterministic_hadamard_matrix  # noqa: E402
from tools.hbm_ceilings import rate  # noqa: E402

HBM_PEAK = 3.35e12


def card():
    name = torch.cuda.get_device_name()
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                               text=True, timeout=30).stdout.strip().splitlines()[torch.cuda.current_device()]
    except Exception as e:  # noqa: BLE001 -- report, do not guess
        power = f"unknown ({e})"
    return name, power


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters


def dense(x, w, precision):
    """the reference's HadamardTransform formula, block-diagonal over the last dimension"""
    n = w.shape[0]
    y = x.to(precision).unflatten(-1, (-1, n)) @ w
    return (y.flatten(-2) / torch.tensor(n, dtype=torch.float64).sqrt()).to(x.dtype)


def within_bound(y, x, w, terms=None):
    """every element within `terms` (log2 n + 1 for a power of two, m + K + 1 with a core) 2^-24 |x_row| of the float64 product, plus
    half an ulp of y's dtype"""
    n = w.shape[0]
    terms = math.log2(n) + 1 if terms is None else terms
    ref = (x.double().unflatten(-1, (-1, n)) @ w.double()) / math.sqrt(n)
    err = (y.double().unflatten(-1, (-1, n)) - ref).abs()
    half_ulp = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11, torch.float32: 0.0}[y.dtype]
    bound = terms * 2.0 ** -24 * x.double().unflatten(-1, (-1, n)).norm(dim=-1, keepdim=True) + half_ulp * ref.abs()
    return bool((err <= bound).all())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--json")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("transform_bench needs a CUDA device")
    gen = torch.Generator(device="cuda").manual_seed(0)
    name, power = card()
    n_copy = 1 << 30
    src = torch.ones(n_copy, dtype=torch.bfloat16, device="cuda")
    dst = torch.empty_like(src)
    copy_gbs = rate(lambda: dst.copy_(src), n_copy * 4)
    del src, dst
    print(f"{name}, power limit / max SM clock: {power}; copy rate {copy_gbs} GB/s")

    cases = []
    x = torch.randn(8192, 4096, device="cuda", generator=gen).bfloat16()
    cases.append(("R1 online [8192, 4096] bf16, n=4096", x, 4096, torch.float32))
    for label, (B, H, S) in (("R3 q prefill [1, 32, 8192, 128]", (1, 32, 8192)), ("R3 k prefill [1, 8, 8192, 128]", (1, 8, 8192)),
                             ("R3 q decode [64, 32, 1, 128]", (64, 32, 1)), ("R3 k decode [64, 8, 1, 128]", (64, 8, 1))):
        cases.append((label, torch.randn(B, S, H, 128, device="cuda", generator=gen).bfloat16().transpose(1, 2), 128, torch.float32))
    w = torch.randn(4096 + 1024 + 1024 + 4096 + 2 * 14336, 4096, device="cuda", generator=gen).bfloat16() * 0.02   # q, k, v, o, gate, up rows
    cases.append(("fp64 fusion of one layer's 4096-input weights (x32 layers)", w, 4096, torch.float64))
    for label, shape, k, m in (("R4 online Llama-3-8B [8192, 14336] bf16, K=224", (8192, 14336), 224, 64),
                               ("R4 online Llama-3-70B [4096, 28672] bf16, K=224", (4096, 28672), 224, 128),
                               ("R4 online Llama-2-7B [8192, 11008] bf16, K=172", (8192, 11008), 172, 64)):
        cases.append((label, torch.randn(*shape, device="cuda", generator=gen).bfloat16(), (k, m), torch.float32))
    cases.append(("fp64 fusion of the 32 down_proj [4096, 14336] of Llama-3-8B, K=224 (x32 layers)",
                  torch.randn(4096, 14336, device="cuda", generator=gen).bfloat16() * 0.02, (224, 64), torch.float64))

    results = []
    for label, t, n, precision in cases:
        if not isinstance(n, int):
            results.append(core_case(label, t, n, precision, a, copy_gbs, gen))
            continue
        h = deterministic_hadamard_matrix(n, precision, "cuda")
        layers = 32 if precision == torch.float64 else 1
        us = timed(lambda: ops.hadamard_transform(t, n, precision=precision), a.iters, a.warmup) * layers
        us_dense = timed(lambda: dense(t, h, precision), max(3, a.iters // 5), 2) * layers
        y = ops.hadamard_transform(t, n, precision=precision)
        ok, ok_dense = within_bound(y, t, h), within_bound(dense(t, h, precision), t, h)
        nbytes = t.numel() * t.element_size() * 2 * layers
        gbs = nbytes / (us * 1e-6) / 1e9
        r = dict(case=label, us=round(us, 1), gbs=round(gbs, 1), of_peak=round(gbs * 1e9 / HBM_PEAK, 3),
                 of_copy=round(gbs / copy_gbs, 3), dense_us=round(us_dense, 1), speedup=round(us_dense / us, 2),
                 kernel_within_bound=ok, dense_within_bound=ok_dense)
        results.append(r)
        print(json.dumps(r))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(card=name, power=power, copy_gbs=copy_gbs, results=results), f, indent=1)


def core_case(label, t, km, precision, a, copy_gbs, gen):
    """one case of order n = K * 2^m: the kernel with a seeded +-1 core against the dense formula with diag(Q) . (C ⊗ H)^T"""
    k, m = km
    n = k * m
    core = (torch.randint(0, 2, (k, k), device="cuda", generator=gen) * 2 - 1).to(torch.int8)
    q = (torch.randint(0, 2, (n,), device="cuda", generator=gen) * 2 - 1).to(torch.int8)
    w = q.to(precision).unsqueeze(1) * torch.kron(core.to(precision), deterministic_hadamard_matrix(m, precision, "cuda")).T
    layers = 32 if precision == torch.float64 else 1
    inverse = precision == torch.float64          # weight_input fusion: value @ M^T
    wd = w.T.contiguous() if inverse else w

    def kernel():
        return ops.hadamard_transform(t, n, q, None, inverse, precision, core=core)

    us = timed(kernel, a.iters, a.warmup) * layers
    us_dense = timed(lambda: dense(t, wd, precision), max(3, a.iters // 10), 1) * layers
    terms = m.bit_length() + k
    ok, ok_dense = within_bound(kernel(), t, wd, terms), within_bound(dense(t, wd, precision), t, wd, terms)
    nbytes = t.numel() * t.element_size() * 2 * layers
    gbs = nbytes / (us * 1e-6) / 1e9
    adds = t.numel() * (k + m.bit_length() - 1) * layers
    compute_us = adds / (33.5e12 if precision == torch.float32 else 17e12) * 1e6
    hbm_us = nbytes / HBM_PEAK * 1e6
    r = dict(case=label, us=round(us, 1), gbs=round(gbs, 1), of_peak=round(gbs * 1e9 / HBM_PEAK, 3), of_copy=round(gbs / copy_gbs, 3),
             hbm_bound_us=round(hbm_us, 1), compute_bound_us=round(compute_us, 1),
             of_bound=round(max(hbm_us, compute_us) / us, 3), dense_us=round(us_dense, 1), speedup=round(us_dense / us, 2),
             kernel_within_bound=ok, dense_within_bound=ok_dense)
    print(json.dumps(r))
    return r


if __name__ == "__main__":
    main()
