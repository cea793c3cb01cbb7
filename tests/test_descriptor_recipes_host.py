"""
Every descriptor the host front end builds, replayed against tests/golden/descriptors.pt.gz (tests/golden/make_golden_descriptors.py):
the per-tensor functions, the observers and the whole-model launches must hand the library the same entry points, arguments and
descriptor fields, and return the same shapes and dtypes or raise the same exceptions, as when the fixture was written.

The fixture predates two deliberate changes, each asserted here rather than regenerated away:
  * descriptors are built by one constructor in which an unnamed field is absent, so the fused observers' descriptors no longer
    carry ctypes' zero (the float32 code) in `seff_dtype`; and the whole-model launches build each module's descriptor with the
    per-tensor recipe, which names the effective scale dtype where the batch left it absent.  The kernels read `seff_dtype` only
    with a global scale or a non-float scale, so neither changes a result.
  * the whole-model launches now run every check of the per-module path, so the inputs below, on which the two disagreed, get
    the per-module outcome; and an NVFP4 module whose non-float scale is divided by its global scale on the host, which the batch
    used to send down the per-module path, is now batched, with the same result.
"""
import copy

import pytest

from compressed_tensors_b200 import _native as N
from tests.golden import load
from tests.golden import make_golden_descriptors as mk

_NI = "NotImplementedError"
_FLOAT_ONLY = "dtype torch.{} is not supported by compressed_tensors_b200 (fp32/fp16/bf16 only)"

# case -> (outcome when the fixture was written, outcome now): the whole-model path used to disagree with the per-module path
DISAGREEMENTS = {
    "batched/pack_f64_weight": (("raise", "ValueError", "batched: tensor 0: the descriptor names no valid dtype for the input"),
                                ("raise", _NI, "input " + _FLOAT_ONLY.format("float64"))),
    "batched/pack_f64_scale": (("raise", "KeyError", "torch.float64"), ("raise", _NI, "scale " + _FLOAT_ONLY.format("float64"))),
    "batched/naive_f64_weight": (("raise", "ValueError", "batched: tensor 0: the descriptor names no valid dtype for the input"),
                                 ("raise", _NI, "input " + _FLOAT_ONLY.format("float64"))),
    "batched/nvfp4_f64_weight": (("raise", "ValueError", "batched: tensor 0: the descriptor names no valid dtype for the input"),
                                 ("raise", _NI, "input " + _FLOAT_ONLY.format("float64"))),
    "batched/pack_float_args": (("ok", None), ("raise", "ValueError", "pack-quantized compression needs integer quantization")),
    "batched/dpack_wide_words": (("raise", "ValueError",
                                  "batched: tensor 0: input holds 80 elements of 4 bytes, the descriptor (8 x 64, 4 bits) needs 64 of 4"),
                                 ("ok", None)),
    "batched/dpack_float_words": (("ok", None), ("raise", "ValueError", "Expected torch.int32 but got torch.float32, Aborting unpack.")),
    "batched/dpack_int_scale": (("ok", None), ("raise", _NI, "scale " + _FLOAT_ONLY.format("int8"))),
    "batched/pack_int_scale": (("ok", None), ("raise", _NI, "scale " + _FLOAT_ONLY.format("int8"))),
    "batched/naive_int_weight": (("ok", None), ("raise", _NI, "input " + _FLOAT_ONLY.format("int8"))),
    "batched/dnaive_int_scale": (("ok", None), ("raise", _NI, "scale " + _FLOAT_ONLY.format("int32"))),
    "batched/dnvfp4_uint8_scale": (("ok", None), ("raise", "ValueError", "stored NVFP4 scales are float8_e4m3fn")),
    "batched/dmxfp4_fp8_scale": (("ok", None), ("raise", "ValueError", "stored MX scales are uint8 exponents")),
}
# case -> (entry points when the fixture was written, entry points now): same outcome and module state, another launch path
LAUNCH_PATH_CHANGES = {
    "batched/nvfp4_int_scale": (("ct_quantize_pack_fp4",), ("ct_host_run_many",)),
}
_FUSED_OBSERVERS = ("ct_observe_quantize_channel", "ct_observe_quantize_pack_int32")
_RECIPE_OPS = (N.OP_QUANTIZE_PACK, N.OP_QUANTIZE, N.OP_DEQUANTIZE)


def _with_seff(desc: tuple, rule) -> tuple:
    fields = dict(desc)
    fields["seff_dtype"] = rule(fields)
    return tuple((f, fields[f]) for f, _ in desc)


def _expected(name: str, rec: dict) -> dict:
    """the fixture's record with the `seff_dtype` changes described above applied"""
    rec = copy.deepcopy(rec)
    calls = []
    for call in rec["calls"]:
        entry, args = call[0], list(call[1:])
        if entry in _FUSED_OBSERVERS:
            args = [("desc", _with_seff(a[1], lambda f: N.DT_NONE if f["seff_dtype"] == 0 else f["seff_dtype"])) if a[0] == "desc" else a
                    for a in args]
        if entry == "ct_host_run_many" and args[0][1] in _RECIPE_OPS:
            args = [("descs", tuple(_with_seff(d, lambda f: f["scale_dtype"] if f["seff_dtype"] == N.DT_NONE else f["seff_dtype"])
                                    for d in a[1])) if a[0] == "descs" else a for a in args]
        calls.append((entry, *args))
    rec["calls"] = tuple(calls)
    return rec


@pytest.fixture(scope="module")
def records():
    return load("descriptors")["cases"], mk.collect()


def test_every_case_is_replayed(records):
    golden, now = records
    assert set(now) == set(golden)


def test_descriptors_match_golden(records):
    golden, now = records
    bad = [name for name in golden if name not in DISAGREEMENTS and name not in LAUNCH_PATH_CHANGES
           and now[name] != _expected(name, golden[name])]
    assert not bad, f"{len(bad)} records differ, first {bad[:5]}"


@pytest.mark.parametrize("name", sorted(DISAGREEMENTS))
def test_whole_model_path_takes_the_per_module_outcome(records, name):
    golden, now = records
    before, after = DISAGREEMENTS[name]
    assert golden[name]["result"] == before
    assert now[name]["result"] == after


@pytest.mark.parametrize("name", sorted(LAUNCH_PATH_CHANGES))
def test_whole_model_path_now_batches(records, name):
    golden, now = records
    before, after = LAUNCH_PATH_CHANGES[name]
    assert tuple(c[0] for c in golden[name]["calls"]) == before
    assert tuple(c[0] for c in now[name]["calls"]) == after
    assert now[name]["result"] == golden[name]["result"] == ("ok", None)
    assert now[name]["modules"] == golden[name]["modules"]
