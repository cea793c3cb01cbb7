#!/usr/bin/env python
"""
Offloaded models on one GPU, with the Linear shapes of a Llama-3-8B decoder layer (q, k, v, o, gate, up, down; bf16):

  (a) forward of a stack of CPU-offloaded layers: every weight is onloaded from pinned host memory (CPUCache, asynchronous copies)
      and used by its Linear.  Reported as onload GB/s against the rate of one pinned H2D copy of the same bytes, measured in the
      same run.
  (b) compress_model W4A16 of a CPU-offloaded and of a disk-offloaded model: the host pipeline (one ct_host_run_many queue for
      the whole model, results written back into the caches) against the per-module path (onload -> kernel -> offload, one
      module at a time).  The two results are compared element by element.
  (c) the same for decompress_model.

Times are CUDA events around whole passes after a warm-up pass on a one-layer model.  Compress / decompress change the model, so
every pass runs on a freshly offloaded copy; each path runs twice, once before and once after the other path, and the faster pass
is reported (both are in the JSON).  The card and its power limit are printed with the numbers.

    python tools/offload_bench.py [--layers 2] [--disk-layers 1] [--iters 3] [--json out.json]
"""
import argparse
import copy
import json
import os
import shutil
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from compressed_tensors_b200.compressors import ModelCompressor, compress_module, decompress_module  # noqa: E402
from compressed_tensors_b200.offload import disable_onloading, offload_module  # noqa: E402
from compressed_tensors_b200.offload.cache import DiskCache  # noqa: E402
from compressed_tensors_b200.quantization import QuantizationConfig, QuantizationStatus, apply_quantization_config  # noqa: E402
from compressed_tensors_b200.quantization.utils import calculate_qparams  # noqa: E402
from tools.dynamic_quant_bench import card, time_call  # noqa: E402

BF = torch.bfloat16
H, I, KV = 4096, 14336, 1024
LAYER = [(H, H), (KV, H), (KV, H), (H, H), (I, H), (I, H), (H, I)]   # (out, in) of q, k, v, o, gate, up, down


def linears(layers: int, seed: int = 0) -> torch.nn.Sequential:
    g = torch.Generator().manual_seed(seed)
    mods = []
    for _ in range(layers):
        for out, inp in LAYER:
            lin = torch.nn.Linear(inp, out, bias=False, dtype=BF)
            lin.weight.data.normal_(0, 0.02, generator=g)
            mods.append(lin)
    return torch.nn.Sequential(*mods)


class Stack(torch.nn.Module):
    """runs every Linear on an input of its own width (the layer's data flow does not matter for onload rates)"""

    def __init__(self, seq):
        super().__init__()
        self.seq = seq

    def forward(self, xs):
        return [lin(xs[lin.in_features]) for lin in self.seq]


def timed(fn):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1e3


def quantized(layers, seed=0):
    model = linears(layers, seed)
    apply_quantization_config(model, QuantizationConfig(config_groups={"W4A16": ["Linear"]}))
    for lin in model:
        args = lin.quantization_scheme.weights
        grp = lin.weight.data.unflatten(-1, (-1, args.group_size))
        s, _ = calculate_qparams(grp.amin(-1), grp.amax(-1), args)
        lin.weight_scale.data.copy_(s.reshape(lin.weight_scale.shape))
        lin.quantization_status = QuantizationStatus.FROZEN
    return model


def offloaded(model, kind, d):
    for m in model:
        offload_module(m, "cuda:0", kind, **({"offload_dir": d} if kind == "disk" else {}))
    return model


def host_values(model):
    out = []
    with disable_onloading():
        for m in model:
            cache = m._parameters
            for k in sorted(cache.offloaded_values):
                v = cache.offloaded_values[k]
                if v is not None:
                    out.append(cache.read(v, "cpu") if isinstance(cache, DiskCache) else v)
    return out


def equal(a, b):
    return len(a) == len(b) and all(x.dtype == y.dtype and x.shape == y.shape and torch.equal(x.view(torch.uint8), y.view(torch.uint8))
                                    for x, y in zip(a, b))


def leg_forward(layers, iters):
    stack = Stack(offloaded(linears(layers), "cpu", None))
    nbytes = sum(lin.in_features * lin.out_features * 2 for lin in stack.seq)
    xs = {w: torch.randn(16, w, dtype=BF, device="cuda") for w in (H, I)}
    with torch.no_grad():
        fwd_us = time_call(lambda: stack(xs), iters, 1)
    src = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    dst = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    copy_us = time_call(lambda: dst.copy_(src, non_blocking=True), iters, 1)
    return dict(layers=layers, bytes=nbytes, forward_ms=fwd_us / 1e3, onload_gbs=nbytes / fwd_us / 1e3,
                pinned_h2d_gbs=nbytes / copy_us / 1e3)


def leg_codec(kind, layers):
    """both paths twice on freshly offloaded copies, in both orders (pipeline first, then per-module first), so that neither
    always runs on host blocks the other has just returned to the caching allocator; the faster of each path's two passes is
    reported, with both passes"""
    base = quantized(layers)
    d = tempfile.mkdtemp(prefix="ct_offload_bench_")
    passes = {"pipeline": {"compress": [], "decompress": []}, "per_module": {"compress": [], "decompress": []}}
    same_c = same_d = True
    try:
        mc = ModelCompressor.from_pretrained_model(base)
        for path in ("pipe", "module"):   # warm-up: one layer each way
            w = offloaded(quantized(1, seed=1), kind, d)
            (mc.compress_model(w) if path == "pipe" else [compress_module(m) for m in w])
            (mc.decompress_model(w) if path == "pipe" else [decompress_module(m) for m in w])
        run = {"pipeline": (lambda mdl: mc.compress_model(mdl), lambda mdl: mc.decompress_model(mdl)),
               "per_module": (lambda mdl: [compress_module(m) for m in mdl], lambda mdl: [decompress_module(m) for m in mdl])}
        for order in (("pipeline", "per_module"), ("per_module", "pipeline")):
            models = {p: offloaded(copy.deepcopy(base), kind, d) for p in order}
            for p in order:
                passes[p]["compress"].append(timed(lambda: run[p][0](models[p])))
            same_c &= equal(host_values(models["pipeline"]), host_values(models["per_module"]))
            for p in order:
                passes[p]["decompress"].append(timed(lambda: run[p][1](models[p])))
            same_d &= equal(host_values(models["pipeline"]), host_values(models["per_module"]))
            del models
    finally:
        shutil.rmtree(d, ignore_errors=True)
    nbytes = sum(m.in_features * m.out_features * 2 for m in base)
    out = dict(kind=kind, layers=layers, bf16_bytes=nbytes)
    for leg, same in (("compress", same_c), ("decompress", same_d)):
        pt, mt = min(passes["pipeline"][leg]), min(passes["per_module"][leg])
        out[leg] = dict(pipeline_s=pt, per_module_s=mt, pipeline_gbs=nbytes / pt / 1e9, per_module_gbs=nbytes / mt / 1e9,
                        pipeline_passes_s=passes["pipeline"][leg], per_module_passes_s=passes["per_module"][leg], outputs_equal=same)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=2)
    ap.add_argument("--disk-layers", type=int, default=1)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    name, power = card()
    print(f"{name}, power limit / max SM clock: {power}")
    res = dict(card=name, power=power, forward=leg_forward(a.layers, a.iters),
               cpu=leg_codec("cpu", a.layers), disk=leg_codec("disk", a.disk_layers))
    f = res["forward"]
    print(f"(a) forward, {f['layers']} CPU-offloaded layers ({f['bytes'] / 1e9:.2f} GB): {f['forward_ms']:.1f} ms, onload "
          f"{f['onload_gbs']:.1f} GB/s; pinned H2D copy {f['pinned_h2d_gbs']:.1f} GB/s")
    for kind in ("cpu", "disk"):
        r = res[kind]
        for leg in ("compress", "decompress"):
            x = r[leg]
            print(f"({'b' if leg == 'compress' else 'c'}) {leg} W4A16, {kind}-offloaded, {r['layers']} layers: pipeline "
                  f"{x['pipeline_s'] * 1e3:.0f} ms ({x['pipeline_gbs']:.2f} GB/s of bf16), per-module {x['per_module_s'] * 1e3:.0f} ms "
                  f"({x['per_module_gbs']:.2f} GB/s); passes (s) pipeline {[round(v, 3) for v in x['pipeline_passes_s']]}, per-module "
                  f"{[round(v, 3) for v in x['per_module_passes_s']]}; outputs equal: {x['outputs_equal']}")
    if a.json:
        with open(a.json, "w") as fh:
            json.dump(res, fh, indent=1)
    ok = all(res[k][leg]["outputs_equal"] for k in ("cpu", "disk") for leg in ("compress", "decompress"))
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
