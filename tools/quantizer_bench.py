#!/usr/bin/env python
"""
CompressedTensorsQuantizer measurements:
  1. the channel observer on wide rows (one thread-block cluster per row) against the unfused path (torch min / max ->
     calculate_qparams -> quantize) at [8192, 28672] and [16384, 53248] bf16, int8 and fp8 codes, as a share of the HBM copy rate
     of tools/hbm_ceilings.py measured in the same run (bytes: weight read once, codes and scales written once);
  2. convert_checkpoint of a synthetic multi-shard bf16 checkpoint on local disk (FP8_DYNAMIC and W4A16) in input GB/s, set
     against a plain read of every byte of the same files (readinto a host buffer), with each shard job's time split into the
     load to the device (safetensors read + H2D, synchronised), process (CUDA events around CompressedTensorsQuantizer.process:
     the kernels), save_file, and the rest (D2H copies and bookkeeping).  The files are freshly written, so both the plain read
     and the conversion read from the page cache.
Every fused result is checked bit for bit against the unfused one.  The card, its power limit and max SM clock are printed with
the numbers.

    python tools/quantizer_bench.py [--shards 4] [--shard-gb 2] [--json out.json]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from compressed_tensors_b200 import ops  # noqa: E402
from compressed_tensors_b200.entrypoints.convert import CompressedTensorsQuantizer, convert_checkpoint  # noqa: E402
from compressed_tensors_b200.quantization import calculate_qparams, preset_name_to_scheme  # noqa: E402
from tools.dynamic_quant_bench import card, time_call  # noqa: E402
from tools.hbm_ceilings import rate  # noqa: E402


def unfused(x, args):
    scale, zp = calculate_qparams(x.amin(-1, keepdim=True), x.amax(-1, keepdim=True), args)
    return ops.quantize(x, scale, None, args, dtype=args.pytorch_dtype()), scale


def kernels(out):
    n = 1 << 30
    a = torch.ones(n, dtype=torch.bfloat16, device="cuda")
    b = torch.empty_like(a)
    copy = rate(lambda: b.copy_(a), n * 4)
    del a, b
    out["hbm_copy_GBps"] = copy
    rows = []
    for shape in ((8192, 28672), (16384, 53248)):
        x = torch.randn(shape, device="cuda", dtype=torch.bfloat16)
        for preset in ("W8A8", "FP8_DYNAMIC"):
            args = preset_name_to_scheme(preset, ["Linear"]).weights
            fq, fs, _ = ops.observe_quantize(x, args)
            uq, us = unfused(x, args)
            assert torch.equal(fq.view(torch.uint8), uq.view(torch.uint8)) and torch.equal(fs, us), (shape, preset)
            nbytes = x.numel() * 3 + shape[0] * 2
            t_f = time_call(lambda: ops.observe_quantize(x, args), 20, 3)
            t_u = time_call(lambda: unfused(x, args), 20, 3)
            gbps = nbytes / (t_f * 1e-6) / 1e9
            rows.append(dict(shape=list(shape), preset=preset, fused_us=round(t_f, 1), unfused_us=round(t_u, 1), fused_GBps=round(gbps, 1),
                             share_of_copy=round(gbps / copy, 3), speedup=round(t_u / t_f, 2)))
            print(rows[-1], flush=True)
        del x
    out["wide_rows"] = rows


class Timed(CompressedTensorsQuantizer):
    """process() with CUDA events around it: the kernels' time per shard (the job's stream)"""
    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.kernel_ms = []

    def process(self, tensors):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        res = super().process(tensors)
        e1.record()
        e1.synchronize()
        self.kernel_ms.append(e0.elapsed_time(e1))
        return res


def _timed(phases: dict, key: str, fn, sync: bool = False):
    """fn with its host wall time added to phases[key] (after a device synchronise when `sync`: the call may return early)"""
    def call(*a, **k):
        t0 = time.perf_counter()
        r = fn(*a, **k)
        if sync:
            torch.cuda.synchronize()
        phases[key] = phases.get(key, 0.0) + time.perf_counter() - t0
        return r
    return call


def plain_read(paths, total):
    """every byte of every file read into one preallocated host buffer (readinto: nothing is left mapped and untouched)"""
    buf = bytearray(max(os.path.getsize(p) for p in paths))
    view = memoryview(buf)
    t0 = time.perf_counter()
    for p in paths:
        with open(p, "rb", buffering=0) as fh:
            n, size = 0, os.path.getsize(p)
            while n < size:
                n += fh.readinto(view[n:size])
    return total / (time.perf_counter() - t0) / 1e9


def checkpoint(out, shards, shard_gb, workdir):
    from safetensors.torch import save_file

    import importlib

    cc_mod = importlib.import_module("compressed_tensors_b200.entrypoints.convert.convert_checkpoint")   # the modules, not the
    cf_mod = importlib.import_module("compressed_tensors_b200.entrypoints.convert.convert_file")         # functions of that name

    src = os.path.join(workdir, "src")
    os.makedirs(src)
    per = int(shard_gb * (1 << 30)) // (2 * 4096 * 14336)   # [14336, 4096] weights per shard
    weight_map, total = {}, 0
    for s in range(shards):
        f = f"model-{s + 1:05d}-of-{shards:05d}.safetensors"
        t = {f"model.layers.{s * per + i}.mlp.up_proj.weight": torch.randn(14336, 4096, dtype=torch.bfloat16) for i in range(per)}
        save_file(t, os.path.join(src, f))
        weight_map.update({k: f for k in t})
        total += sum(v.nbytes for v in t.values())
    with open(os.path.join(src, "model.safetensors.index.json"), "w") as fh:
        json.dump({"metadata": {"total_size": total}, "weight_map": weight_map}, fh)
    with open(os.path.join(src, "config.json"), "w") as fh:
        json.dump({"model_type": "llama"}, fh)
    paths = [os.path.join(src, f) for f in sorted(set(weight_map.values()))]
    out["checkpoint"] = dict(shards=shards, input_GB=round(total / 1e9, 2), plain_read_GBps=round(plain_read(paths, total), 2), runs=[])
    print(out["checkpoint"], flush=True)
    for preset in ("FP8_DYNAMIC", "W4A16"):   # first calls (module load, allocator) outside the timed runs
        Timed(preset).process({"w.weight": torch.randn(14336, 4096, dtype=torch.bfloat16, device="cuda")})
    load, save, convert = cf_mod.load_tensors_from_inverse_weight_map, cf_mod.save_file, cc_mod.convert_file
    try:
        for preset in ("FP8_DYNAMIC", "W4A16"):
            for workers in (1, 2):
                phases = {}
                cf_mod.load_tensors_from_inverse_weight_map = _timed(phases, "load_to_device_s", load, sync=True)
                cf_mod.save_file = _timed(phases, "save_file_s", save)
                cc_mod.convert_file = _timed(phases, "shard_job_s", convert)
                conv = Timed(preset)
                dst = os.path.join(workdir, f"out-{preset}-{workers}")
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                convert_checkpoint(src, dst, conv, max_workers=workers, device="cuda")
                wall = time.perf_counter() - t0
                kern = sum(conv.kernel_ms) / 1e3
                phases = {k: round(v, 2) for k, v in phases.items()}
                phases["process_s"] = round(kern, 2)
                phases["d2h_and_rest_s"] = round(phases["shard_job_s"] - phases["load_to_device_s"] - kern - phases["save_file_s"], 2)
                run = dict(preset=preset, workers=workers, wall_s=round(wall, 2), input_GBps=round(total / wall / 1e9, 2),
                           kernel_ms_per_shard=[round(m, 1) for m in conv.kernel_ms], kernel_share_of_wall=round(kern / wall, 3),
                           phase_seconds_summed_over_jobs=phases)
                out["checkpoint"]["runs"].append(run)
                print(run, flush=True)
    finally:
        cf_mod.load_tensors_from_inverse_weight_map, cf_mod.save_file, cc_mod.convert_file = load, save, convert


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shards", type=int, default=4)
    ap.add_argument("--shard-gb", type=float, default=2.0)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    name, power = card()
    out = {"card": name, "power_limit_and_max_sm_clock": power}
    print(out, flush=True)
    kernels(out)
    with tempfile.TemporaryDirectory() as d:
        checkpoint(out, a.shards, a.shard_gb, d)
    print(json.dumps(out))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
