"""Offload caches, module offloading and dispatch on the CPU: cache semantics, the disk round trip, restoring a module, the direct
state-dict helpers on offloaded modules, and the entry points that stay refused."""
import pytest
import torch

from compressed_tensors_b200.offload import (OffloadCache, align_module_device, disable_offloading, disable_onloading, dispatch_with_map,
                                             from_accelerate, get_cache_init_kwargs, get_device_map, get_execution_device,
                                             get_offloaded_device, load_offloaded_model, offload_module, register_offload_module,
                                             remove_dispatch, remove_module_offload, set_onload_device, to_accelerate, to_meta,
                                             unwrap_offload_forward, update_offload_parameter)
from compressed_tensors_b200.offload.cache import CPUCache, DeviceCache, DiskCache
from compressed_tensors_b200.offload.dispatch import dispatch_model
from compressed_tensors_b200.offload.utils import get_module_sizes, module_size, send_tensors
from compressed_tensors_b200.utils.module import get_direct_state_dict, replace_direct_state_dict


def _linear(seed=0, bias=True):
    torch.manual_seed(seed)
    return torch.nn.Linear(8, 4, bias=bias)


def test_cls_from_device():
    assert OffloadCache.cls_from_device("cpu") is CPUCache
    assert OffloadCache.cls_from_device(torch.device("cpu")) is CPUCache
    assert OffloadCache.cls_from_device("disk") is DiskCache
    assert OffloadCache.cls_from_device("cuda:0") is DeviceCache
    with pytest.raises(NotImplementedError):
        OffloadCache.cls_from_device("meta")


def test_cpu_cache_offload_on_set_onload_on_get():
    cache = CPUCache("cpu")
    t = torch.arange(6, dtype=torch.float32)
    cache["x"] = t
    assert "x" in cache and len(cache) == 1 and list(cache) == ["x"]
    assert torch.equal(cache["x"], t)
    assert cache.offloaded_values["x"].device.type == "cpu"
    del cache["x"]
    assert "x" not in cache and len(cache) == 0


def test_disable_onloading_assigns_and_reads_directly():
    cache = CPUCache("cpu")
    t = torch.ones(3)
    with disable_onloading():
        cache["x"] = t
        assert cache.offloaded_values["x"] is t
        assert cache["x"] is t
        with disable_onloading():   # nested: still disabled
            assert OffloadCache.onloading_disabled
        assert OffloadCache.onloading_disabled
    assert not OffloadCache.onloading_disabled


def test_disable_offloading_keeps_onloaded_values_until_exit():
    cache = DeviceCache("cpu")   # a "device" cache on the CPU: onload returns the offloaded tensor
    cache["x"] = torch.ones(3)

    class Counting(CPUCache):
        calls = 0

        def onload(self, offloaded):
            Counting.calls += 1
            return offloaded.clone()

    c = Counting("cpu")
    c["x"] = torch.ones(3)
    first = c["x"]
    assert c["x"] is not first and Counting.calls == 2
    with disable_offloading():
        a = c["x"]
        assert c["x"] is a and Counting.calls == 3
        with disable_offloading():
            assert c["x"] is a
        assert len(OffloadCache.keep_onloaded_values) == 1
    assert len(OffloadCache.keep_onloaded_values) == 0
    assert not OffloadCache.offloading_disabled


def test_update_in_place_updates_kept_copy():
    class Cloning(CPUCache):
        def onload(self, offloaded):
            return offloaded.clone()

    c = Cloning("cpu")
    c["x"] = torch.zeros(4)
    offloaded = c.offloaded_values["x"]
    with disable_offloading():
        kept = c["x"]
        c["x"] = torch.full((4,), 7.0)
        assert c.offloaded_values["x"] is offloaded   # same shape: written in place
        assert torch.equal(offloaded, torch.full((4,), 7.0))
        assert torch.equal(kept, torch.full((4,), 7.0))
    c["x"] = torch.ones(2)   # new shape: a new offloaded tensor
    assert c.offloaded_values["x"] is not offloaded and torch.equal(c["x"], torch.ones(2))
    c["y"] = None
    assert c["y"] is None


def test_disk_cache_round_trip(tmp_path):
    cache = DiskCache("cpu", offload_dir=str(tmp_path))
    t = torch.randn(5, 3, dtype=torch.bfloat16)
    cache["w"] = t
    off = cache.offloaded_values["w"]
    assert off.device.type == "meta" and off.shape == t.shape and off.dtype == t.dtype
    files = list(tmp_path.iterdir())
    assert len(files) == 1 and files[0].name.startswith("ct_disk_cache") and files[0].suffix == ".safetensors"
    assert torch.equal(cache["w"], t)
    cache["w"] = torch.zeros(5, 3, dtype=torch.bfloat16)   # update rewrites the same file
    assert cache.offloaded_values["w"] is off and list(tmp_path.iterdir()) == files
    assert torch.equal(cache["w"], torch.zeros(5, 3, dtype=torch.bfloat16))
    with disable_onloading():
        assert cache["w"] is off
    del cache["w"]
    assert list(tmp_path.iterdir()) == [] and off not in DiskCache.index
    with pytest.raises(ValueError, match="offload_dir"):
        DiskCache("cpu")


def test_offload_module_and_remove_restore_forward_and_dicts(tmp_path):
    for device, kwargs in (("cpu", {}), ("disk", {"offload_dir": str(tmp_path)})):
        lin = _linear()
        ref = _linear()
        forward = lin.forward
        offload_module(lin, "cpu", device, **kwargs)
        assert isinstance(lin._parameters, OffloadCache) and isinstance(lin._buffers, OffloadCache)
        assert get_execution_device(lin) == "cpu" and str(get_offloaded_device(lin)) == device
        with pytest.raises(ValueError, match="twice"):
            offload_module(lin, "cpu", device, **kwargs)
        x = torch.randn(2, 8)
        assert torch.equal(lin(x), ref(x))
        remove_module_offload(lin, onload_tensors=True)
        assert type(lin._parameters) is dict and type(lin._buffers) is dict
        assert lin.forward == forward and not hasattr(lin, "_original_forward_func")
        assert torch.equal(lin.weight, ref.weight) and isinstance(lin.weight, torch.nn.Parameter)
        assert torch.equal(lin(x), ref(x))


def test_unwrap_offload_forward_rewraps_replaced_forward():
    lin = _linear()
    offload_module(lin, "cpu", "cpu")
    with unwrap_offload_forward(lin):
        inner = lin.forward.__func__

        def doubled(self, x):
            return inner(self, x) * 2

        lin.forward = doubled.__get__(lin)
    x = torch.randn(1, 8)
    assert torch.equal(lin(x), _linear()(x) * 2)
    remove_module_offload(lin)
    assert torch.equal(lin(x), _linear()(x) * 2)


def test_direct_state_dict_on_offloaded_modules(tmp_path):
    for device, kwargs in (("cpu", {}), ("disk", {"offload_dir": str(tmp_path)})):
        lin = _linear()
        offload_module(lin, "cpu", device, **kwargs)
        sd = get_direct_state_dict(lin)
        assert set(sd) == {"weight", "bias"} and torch.equal(sd["weight"], _linear().weight)
        replace_direct_state_dict(lin, {"weight_packed": torch.ones(4, 2, dtype=torch.int32), "bias": sd["bias"]})
        assert set(lin._parameters) == {"weight_packed", "bias"}
        assert isinstance(lin._parameters, OffloadCache)
        assert torch.equal(lin.weight_packed, torch.ones(4, 2, dtype=torch.int32))
        assert isinstance(lin.weight_packed, torch.nn.Parameter) and not lin.weight_packed.requires_grad
        with disable_onloading():
            kept = lin._parameters["weight_packed"]
            if device == "disk":
                assert kept.device.type == "meta"
            else:
                assert kept.device.type == "cpu"
        to_meta(lin)
        with disable_onloading():
            assert all(v.device.type == "meta" for v in lin._parameters.values())
        remove_module_offload(lin)


def test_update_offload_parameter_and_align(tmp_path):
    lin = _linear()
    offload_module(lin, "cpu", "disk", offload_dir=str(tmp_path))
    update_offload_parameter(lin, "weight", torch.zeros(4, 8))
    assert torch.equal(lin.weight, torch.zeros(4, 8))
    with pytest.raises(AttributeError):
        update_offload_parameter(lin, "nope", torch.zeros(1))
    with align_module_device(lin):
        w = lin.weight
        assert lin.weight is w   # kept onloaded
    plain = _linear()
    with align_module_device(plain, "cpu"):
        assert plain.weight.device.type == "cpu"
    update_offload_parameter(plain, "bias", torch.ones(4))
    assert torch.equal(plain.bias, torch.ones(4))


def test_register_offload_module_and_cache_kwargs(tmp_path):
    parent = torch.nn.Sequential(_linear())
    offload_module(parent[0], "cpu", "disk", offload_dir=str(tmp_path))
    kw = get_cache_init_kwargs(parent[0])
    assert kw["onload_device"] == "cpu" and kw["offload_device"] == "disk" and str(kw["offload_dir"]) == str(tmp_path.resolve())
    child = _linear(1)
    register_offload_module(parent[0], "child", child)
    assert isinstance(child._parameters, DiskCache) and parent[0].child is child


def test_set_onload_device_dispatch_map_and_remove(tmp_path):
    model = torch.nn.Sequential(_linear(0), _linear(1, bias=False))
    ref = torch.nn.Sequential(_linear(0), _linear(1, bias=False))
    x = torch.randn(2, 8)
    set_onload_device(model, "cpu")
    assert all(isinstance(m._parameters, CPUCache) for m in model.modules())
    assert torch.equal(model[0](x), ref[0](x))
    dmap = get_device_map(model)
    assert set(dmap) == {"", "0", "1"} and all(v == ("cpu", torch.device("cpu")) for v in dmap.values())
    remove_dispatch(model)
    assert all(type(m._parameters) is dict for m in model.modules())
    dispatch_with_map(model, {"0": ("cpu", "disk"), "1": ("cpu", None), "missing": ("cpu", "cpu")}, offload_dir=str(tmp_path),
                      show_progress=False)
    assert isinstance(model[0]._parameters, DiskCache) and type(model[1]._parameters) is dict
    assert torch.equal(model[0](x), ref[0](x))
    remove_dispatch(model, onload_tensors=True)


def test_dispatch_model_sizes_and_cpu_fallback():
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(8, 4), torch.nn.Linear(4, 8))
    sizes = get_module_sizes(model)
    assert [m for m, _ in sizes] == [model[0], model[1]] and all(s == module_size(m) for m, s in sizes)
    x = torch.randn(2, 8)
    expect = model(x)
    # "cpu" as the only device: every module onloads to and offloads to the CPU
    dispatch_model(model, device_memory={torch.device("cpu"): 10 ** 6}, extra_memory=0)
    assert all(isinstance(m._parameters, CPUCache) and get_execution_device(m) == torch.device("cpu") for m in model)
    assert torch.equal(model(x), expect)
    # too little room for even one module plus the reserve
    with pytest.raises(ValueError, match="Cannot fit"):
        dispatch_model(model, device_memory={torch.device("cpu"): module_size(model[0]) - 1}, extra_memory=0)


def test_send_tensors_nested():
    t = torch.ones(2)
    out = send_tensors({"a": [t, (t,)], "b": 3}, device="cpu")
    assert out["a"][0] is t and out["a"][1][0] is t and out["b"] == 3
    p = torch.nn.Parameter(torch.ones(2))
    p.extra = 5
    m = send_tensors(p, dtype=torch.float64)
    assert isinstance(m, torch.nn.Parameter) and m.dtype == torch.float64 and m.extra == 5


@pytest.mark.parametrize("fn,name", [(load_offloaded_model, "load_offloaded_model"), (from_accelerate, "from_accelerate"),
                                     (to_accelerate, "to_accelerate")])
def test_refused_entry_points_name_themselves(fn, name):
    with pytest.raises(NotImplementedError, match=name):
        fn(torch.nn.Linear(2, 2))


def test_distributed_caches_refused(monkeypatch):
    import torch.distributed as dist

    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    for device, name in (("cpu", "dist_cpu"), ("disk", "dist_disk"), ("cuda", "dist_device")):
        with pytest.raises(NotImplementedError, match=name):
            OffloadCache.cls_from_device(device)


def test_unchanged_buffer_of_a_disk_offloaded_module_stays_a_buffer(tmp_path):
    lin = _linear()
    lin.register_buffer("scale", torch.full((4,), 3.0))
    offload_module(lin, "cpu", "disk", offload_dir=str(tmp_path))
    with disable_onloading():
        kept = lin._buffers.offloaded_values["scale"]
    path = DiskCache.index[kept]["safetensors_file"]
    sd = get_direct_state_dict(lin)
    replace_direct_state_dict(lin, {"weight": sd["weight"] * 2, "bias": sd["bias"], "scale": kept})
    assert "scale" in lin._buffers and "scale" not in lin._parameters
    assert lin._buffers.offloaded_values["scale"] is kept and kept in DiskCache.index
    assert torch.equal(lin.scale, torch.full((4,), 3.0)) and torch.equal(lin.weight, _linear().weight * 2)
    import os

    assert os.path.exists(path)
