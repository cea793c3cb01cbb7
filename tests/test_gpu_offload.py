"""
Offloading on the H100: the caches onloading to the device (pinned host memory, asynchronous copies, the event that guards an
update against a copy in flight), dispatch and module offloading, a seeded 2-layer Llama run CPU-offloaded, disk-offloaded and
dispatched against the same model on the GPU, compress_model / decompress_model of offloaded models through one host pipeline
queue against a GPU-resident copy, and transform fusion on an offloaded model.
"""
import copy

import pytest
import torch

from compressed_tensors_b200 import ops
from compressed_tensors_b200.offload import (OffloadCache, align_module_device, disable_offloading, disable_onloading, dispatch_model,
                                             dispatch_with_map, get_execution_device, offload_module, remove_dispatch,
                                             remove_module_offload, set_onload_device, update_offload_parameter)
from compressed_tensors_b200.offload.cache import CPUCache, DeviceCache, DiskCache

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
BF = torch.bfloat16


# ---- caches ------------------------------------------------------------------------------------------------------------------
def test_cpu_cache_pins_and_onloads_asynchronously():
    cache = CPUCache(DEV)
    src = torch.randn(256, 512, dtype=BF)
    cache["w"] = src
    off = cache.offloaded_values["w"]
    assert off.device.type == "cpu" and off.is_pinned() and torch.equal(off, src)
    pinned = torch.randn(8).pin_memory()
    cache["p"] = pinned
    assert cache.offloaded_values["p"] is pinned   # already pinned: kept as it is
    on = cache["w"]
    assert on.device == DEV and torch.equal(on.cpu(), src)
    cache["g"] = torch.ones(4, device=DEV)         # offload from the device
    assert cache.offloaded_values["g"].is_pinned() and torch.equal(cache["g"].cpu(), torch.ones(4))
    p = torch.nn.Parameter(torch.ones(3), requires_grad=False)
    cache["param"] = p
    assert isinstance(cache["param"], torch.nn.Parameter) and cache["param"].device == DEV


def test_onload_then_update_reads_no_stale_bytes():
    """an onload still in flight when the same tensor is updated from host memory: the copy sees the old bytes, every later read
    the new ones"""
    lin = torch.nn.Linear(8192, 8192, bias=False, dtype=BF)   # 128 MiB: the H2D copy is still running when the update starts
    old = lin.weight.detach().clone()
    offload_module(lin, DEV, "cpu")
    new = torch.randn_like(old)
    for _ in range(3):
        onloaded = lin.weight
        update_offload_parameter(lin, "weight", new)
        torch.cuda.synchronize()
        assert torch.equal(onloaded.cpu(), old)
        assert torch.equal(lin.weight.cpu(), new)
        update_offload_parameter(lin, "weight", old)
    with disable_offloading():
        kept = lin.weight
        update_offload_parameter(lin, "weight", new)
        assert torch.equal(kept.cpu(), new)   # the kept onloaded copy follows the update


def test_device_cache_and_disk_cache_onload_to_device(tmp_path):
    dc = DeviceCache(DEV)
    t = torch.randn(16, 16)
    dc["x"] = t
    assert dc.offloaded_values["x"].device == DEV and dc["x"] is dc.offloaded_values["x"]
    assert DeviceCache("cuda:0", "cpu").offload_device == torch.device("cpu")
    disk = DiskCache(DEV, offload_dir=str(tmp_path))
    disk["x"] = t
    assert disk.offloaded_values["x"].device.type == "meta"
    got = disk["x"]
    assert got.device == DEV and torch.equal(got.cpu(), t)
    disk["x"] = t.to(DEV) * 2
    assert torch.equal(disk["x"].cpu(), t * 2)
    with disable_onloading():
        assert disk["x"].device.type == "meta"


def test_module_forward_moves_inputs_and_align(tmp_path):
    torch.manual_seed(0)
    for offload, kw in (("cpu", {}), ("disk", {"offload_dir": str(tmp_path)}), ("cuda:0", {})):
        lin = torch.nn.Linear(64, 32)
        ref = copy.deepcopy(lin).to(DEV)
        offload_module(lin, DEV, offload, **kw)
        x = torch.randn(4, 64)
        y = lin(x)   # a CPU input follows the weights to the device
        assert y.device == DEV and torch.equal(y, ref(x.to(DEV)))
        assert get_execution_device(lin) == DEV
        with align_module_device(lin):
            assert lin.weight is lin.weight and lin.weight.device == DEV
        with align_module_device(lin, "cpu"):
            assert lin.weight.device.type == "cpu"
        remove_module_offload(lin, onload_tensors=True)
        assert lin.weight.device == DEV and torch.equal(lin.weight, ref.weight)


def test_dispatch_model_on_the_gpu():
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(256, 256), torch.nn.Linear(256, 256))
    x = torch.randn(2, 256)
    expect = copy.deepcopy(model).to(DEV)(x.to(DEV))
    dispatch_model(model)
    assert all(isinstance(m._parameters, DeviceCache) and m._parameters.offload_device == DEV for m in model)
    assert torch.equal(model(x), expect)
    # no room: the whole model is CPU-offloaded and onloaded to the device
    dispatch_model(model, device_memory={DEV: 1 << 20}, extra_memory=1 << 19)
    assert all(isinstance(m._parameters, CPUCache) and m._parameters.onload_device == DEV for m in model)
    assert torch.equal(model(x), expect)
    remove_dispatch(model)


# ---- a 2-layer Llama -----------------------------------------------------------------------------------------------------------
def _llama():
    from transformers import LlamaConfig, LlamaForCausalLM

    torch.manual_seed(1234)
    cfg = LlamaConfig(num_hidden_layers=2, hidden_size=256, num_attention_heads=4, num_key_value_heads=2, head_dim=64, vocab_size=256,
                      intermediate_size=512, max_position_embeddings=128)
    return LlamaForCausalLM(cfg).to(BF).eval()


@pytest.mark.parametrize("how", ["cpu", "disk", "dispatch"])
def test_llama_forward_offloaded_equals_on_gpu(how, tmp_path):
    model = _llama()
    on_gpu = copy.deepcopy(model).to(DEV)
    ids = torch.randint(0, 256, (2, 16), generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        want = on_gpu(ids.to(DEV), use_cache=False).logits
    if how == "cpu":
        set_onload_device(model, DEV)
        assert isinstance(model.model.layers[0].mlp.down_proj._parameters, CPUCache)
    elif how == "disk":
        dispatch_with_map(model, {n: (DEV, "disk") for n, _ in model.named_modules()}, offload_dir=str(tmp_path), show_progress=False)
        assert isinstance(model.model.layers[0].mlp.down_proj._parameters, DiskCache)
    else:
        dispatch_model(model)
    with torch.no_grad():
        got = model(ids, use_cache=False).logits
    assert torch.equal(got, want)


# ---- compress / decompress offloaded models ------------------------------------------------------------------------------------
def _quantized_model(preset):
    """three Linears with the preset's weight scheme and observed qparams, on the CPU"""
    from compressed_tensors_b200.quantization import QuantizationConfig, QuantizationStatus, apply_quantization_config
    from compressed_tensors_b200.quantization.utils import calculate_qparams, generate_gparam

    torch.manual_seed(9)
    model = torch.nn.Sequential(torch.nn.Linear(1024, 512, bias=False), torch.nn.Linear(512, 1536, bias=False),
                                torch.nn.Linear(1536, 512, bias=False)).to(BF)
    apply_quantization_config(model, QuantizationConfig(config_groups={preset: ["Linear"]}))
    for lin in model:
        a = lin.quantization_scheme.weights
        w = lin.weight.data
        if a.strategy in ("group", "tensor_group"):
            grp = w.unflatten(-1, (-1, a.group_size))
            mn, mx = grp.amin(-1), grp.amax(-1)
        elif a.strategy == "channel":
            mn, mx = w.amin(-1, keepdim=True), w.amax(-1, keepdim=True)
        else:
            mn, mx = w.min().reshape(1), w.max().reshape(1)
        if hasattr(lin, "weight_global_scale"):
            gs = generate_gparam(w.min(), w.max())
            lin.weight_global_scale.data.copy_(gs)
            s, z = calculate_qparams(mn, mx, a, global_scale=gs)
        else:
            s, z = calculate_qparams(mn, mx, a)
        lin.weight_scale.data = s.to(lin.weight_scale.dtype).reshape(lin.weight_scale.shape)
        if hasattr(lin, "weight_zero_point"):
            lin.weight_zero_point.data = z.to(lin.weight_zero_point.dtype).reshape(lin.weight_zero_point.shape)
        lin.quantization_status = QuantizationStatus.FROZEN
    return model


def _offloaded_state(model):
    with disable_onloading():
        return {f"{i}.{k}": v for i, m in enumerate(model) for k, v in m._parameters.items()}


def _host_state(model, kind):
    """every offloaded tensor's bytes, read on the CPU; checks they are kept where the cache keeps them"""
    out = {}
    for i, m in enumerate(model):
        cache = m._parameters
        assert isinstance(cache, CPUCache if kind == "cpu" else DiskCache)
        for k, v in cache.offloaded_values.items():
            if v is None:   # bias=False: a registered None, absent from state_dict() as well
                continue
            if kind == "cpu":
                assert v.device.type == "cpu" and v.is_pinned(), (i, k)
            else:
                assert v.device.type == "meta", (i, k)
                v = cache.read(v, "cpu")
            out[f"{i}.{k}"] = v.detach()
    return out


def _same_bytes(got: dict, want: dict, what: str):
    assert set(got) == set(want), (what, set(got) ^ set(want))
    for k in want:
        g, w = got[k].cpu(), want[k].cpu()
        assert g.dtype == w.dtype and g.shape == w.shape, (what, k, g.dtype, w.dtype, g.shape, w.shape)
        assert torch.equal(g.contiguous().view(torch.uint8), w.contiguous().view(torch.uint8)), (what, k)


@pytest.mark.parametrize("kind", ["cpu", "disk"])
@pytest.mark.parametrize("preset", ["W4A16", "FP8", "NVFP4A16", "MXFP4A16"])
def test_compress_decompress_offloaded_model_equals_gpu_model(preset, kind, tmp_path, monkeypatch):
    from compressed_tensors_b200.compressors import ModelCompressor

    model = _quantized_model(preset)
    on_gpu = copy.deepcopy(model).to(DEV)
    for m in model:
        offload_module(m, DEV, kind, **({"offload_dir": str(tmp_path)} if kind == "disk" else {}))
    mc = ModelCompressor.from_pretrained_model(on_gpu)

    calls = []
    real = ops.host_batched
    monkeypatch.setattr(ops, "host_batched", lambda op, probs, *a: (calls.append(len(probs)), real(op, probs, *a))[1])

    mc.compress_model(on_gpu)
    mc.compress_model(model)
    assert calls == [3], calls   # the whole offloaded model in one pipeline queue
    want = {f"{i}.{k}": v for i, m in enumerate(on_gpu) for k, v in m.state_dict().items()}
    _same_bytes(_host_state(model, kind), want, f"{preset} {kind} compressed")

    mc.decompress_model(on_gpu)
    mc.decompress_model(model)
    assert calls == [3, 3], calls
    want = {f"{i}.{k}": v for i, m in enumerate(on_gpu) for k, v in m.state_dict().items()}
    _same_bytes(_host_state(model, kind), want, f"{preset} {kind} decompressed")
    if kind == "disk":   # the files of replaced tensors are gone: one file per offloaded tensor
        assert len(list(tmp_path.iterdir())) == len(want)


# ---- transforms -----------------------------------------------------------------------------------------------------------------
def test_transform_fusion_on_cpu_offloaded_model_equals_gpu_model():
    from compressed_tensors_b200.transform import TransformArgs, TransformConfig, TransformScheme, apply_transform_config

    model = _llama()
    on_gpu = copy.deepcopy(model).to(DEV)
    # SpinQuant-like: R1 on the residual stream (embedding out, every reader in, every writer out), R2 per head on v / o
    config = TransformConfig(config_groups={
        "R1": TransformScheme(type="hadamard", apply=[
            TransformArgs(targets=["re:.*embed_tokens$"], location="weight_output"),
            TransformArgs(targets=["re:.*(q|k|v|up|gate)_proj$", "lm_head"], location="weight_input", inverse=True),
            TransformArgs(targets=["re:.*(o|down)_proj$"], location="weight_output"),
        ]),
        "R2": TransformScheme(type="hadamard", head_dim=64, apply=[
            TransformArgs(targets=["re:.*v_proj$"], location="weight_output"),
            TransformArgs(targets=["re:.*o_proj$"], location="weight_input", inverse=True),
        ]),
    })
    set_onload_device(model, DEV)
    apply_transform_config(on_gpu, config)
    apply_transform_config(model, config)
    got = {}
    for name, m in model.named_modules():
        if isinstance(m._parameters, OffloadCache):
            assert isinstance(m._parameters, CPUCache)
            for k, v in m._parameters.offloaded_values.items():
                assert v is None or v.device.type == "cpu"
                if v is not None:
                    got[f"{name}.{k}" if name else k] = v
    want = dict(on_gpu.named_parameters(remove_duplicate=False))
    _same_bytes({k: got[k] for k in want}, want, "fused weights")


# ---- the reference's cache, interface and module cases, restated ---------------------------------------------------------------
def _cache(kind, tmp_path):
    if kind == "cpu":
        return CPUCache(DEV)
    if kind == "device":
        return DeviceCache(DEV)
    return DiskCache(DEV, offload_dir=str(tmp_path))


def _kept_device(kind):
    return {"cpu": "cpu", "device": "cuda", "disk": "meta"}[kind]


CACHES = ["cpu", "device", "disk"]


@pytest.mark.parametrize("kind", CACHES)
def test_cache_onloading_offload_onload(kind, tmp_path):
    cache = _cache(kind, tmp_path)
    t = torch.ones(10)
    cache["weight"] = t
    onloaded = cache["weight"]
    assert type(onloaded) is type(t) and onloaded.device == DEV and torch.equal(onloaded.cpu(), t)
    on_dev = torch.ones(10, device=DEV)
    offloaded = cache.offload(on_dev)
    assert offloaded.device.type == _kept_device(kind)
    back = cache.onload(offloaded)
    assert back.device == DEV and torch.equal(back, on_dev)


@pytest.mark.parametrize("kind", CACHES)
def test_cache_garbage_collect_and_delete(kind, tmp_path):
    import gc
    from weakref import ref

    cache = _cache(kind, tmp_path)
    cache["weight"] = torch.ones(10)
    onloaded = cache["weight"]
    r = ref(onloaded)
    del onloaded
    gc.collect()
    assert kind == "device" or r() is None   # a device cache onloads to the offloaded tensor itself
    onloaded = cache["weight"]
    r = ref(onloaded)
    with disable_offloading():
        del cache["weight"]
        del onloaded
        gc.collect()
        assert kind == "device" or r() is None
    assert "weight" not in cache


@pytest.mark.parametrize("kind", ["cpu", "disk"])
def test_cache_disable_offloading_releases_on_exit(kind, tmp_path):
    import gc
    from weakref import ref

    cache = _cache(kind, tmp_path)
    cache["weight"] = torch.ones(10)
    outside = cache["weight"]
    outside_ref = ref(outside)
    with disable_offloading():
        inside = cache["weight"]
        inside_ref = ref(inside)
        assert inside.device == DEV
        del outside, inside
        gc.collect()
        assert outside_ref() is None and inside_ref() is not None
    gc.collect()
    assert inside_ref() is None


@pytest.mark.parametrize("kind", CACHES)
def test_cache_disable_onloading_and_shared_attributes(kind, tmp_path):
    cache = _cache(kind, tmp_path)
    t = torch.ones(10)
    cache.offloaded_values["weight"] = t
    with disable_onloading():
        assert cache["weight"] is t
    assert cache.offloading_disabled is type(cache).offloading_disabled
    assert cache.onloading_disabled is type(cache).onloading_disabled
    assert cache.keep_onloaded_values is type(cache).keep_onloaded_values
    assert not hasattr(type(cache), "onload_device") and not hasattr(type(cache), "offloaded_values")


@pytest.mark.parametrize("kind", CACHES)
def test_cache_tensor_subclasses_and_update(kind, tmp_path):
    cache = _cache(kind, tmp_path)
    values = {"tensor": torch.ones(10), "param": torch.nn.Parameter(torch.ones(10), requires_grad=False),
              "buffer": torch.nn.Buffer(torch.ones(10))}
    for k, v in values.items():
        cache[k] = v
    for k, v in values.items():
        got = cache[k]
        assert got.device == DEV and torch.equal(got.cpu(), v.detach())
        assert isinstance(got, torch.nn.Parameter) == isinstance(v, torch.nn.Parameter)
        with disable_onloading():
            assert cache[k].device.type == _kept_device(kind)
    cache["tensor"] = torch.full((10,), 2.0, device=DEV)
    assert torch.equal(cache["tensor"].cpu(), torch.full((10,), 2.0))


def test_cpu_cache_logs_memory_hint(monkeypatch, caplog):
    import compressed_tensors_b200.offload.cache.cpu as cpu_mod

    def oom(t):
        raise RuntimeError("mmap failed: Cannot allocate memory")

    monkeypatch.setattr(cpu_mod, "_pinned", oom)
    with caplog.at_level("WARNING"), pytest.raises(RuntimeError, match="Cannot allocate memory"):
        CPUCache(DEV).offload(torch.zeros(1))
    assert any("ran out of host memory" in r.getMessage() for r in caplog.records)


def _linear():
    torch.manual_seed(0)
    return torch.nn.Linear(5, 5)


def test_update_offload_parameter_with_grad():
    lin = _linear()
    zeros = torch.nn.Parameter(torch.zeros(5, 5), requires_grad=True)
    update_offload_parameter(lin, "weight", zeros)
    assert torch.equal(lin.weight.detach(), zeros.detach())
    ones = torch.nn.Parameter(torch.ones(5, 5), requires_grad=True)
    offload_module(lin, DEV, "cpu")
    update_offload_parameter(lin, "weight", ones)
    assert lin.weight.device == DEV and torch.equal(lin.weight.cpu(), ones.detach())


def test_cache_kwargs_and_register_offload_module(tmp_path):
    from compressed_tensors_b200.offload import get_cache_init_kwargs, get_cache_kwargs, register_offload_module

    lin = _linear()
    with pytest.warns(DeprecationWarning):
        assert get_cache_kwargs(lin) == {} and get_cache_kwargs(lin, default={"custom": "value"}) == {"custom": "value"}
    assert get_cache_init_kwargs(lin) == {"onload_device": torch.device("cpu"), "offload_device": torch.device("cpu")}
    offload_module(lin, DEV, "cpu")
    with pytest.warns(DeprecationWarning):
        assert get_cache_kwargs(lin) == {}
    assert get_cache_init_kwargs(lin) == {"onload_device": DEV, "offload_device": torch.device("cpu")}
    child = torch.nn.Linear(5, 5)
    register_offload_module(lin, "child", child)
    assert isinstance(child._parameters, CPUCache) and child._parameters.onload_device == DEV
    disk = _linear()
    offload_module(disk, DEV, "disk", offload_dir=str(tmp_path))
    with pytest.warns(DeprecationWarning):
        assert get_cache_kwargs(disk) == {"offload_dir": tmp_path.resolve()}
    kw = get_cache_init_kwargs(disk)
    assert kw["offload_device"] == "disk" and kw["offload_dir"] == tmp_path.resolve()
    child = torch.nn.Linear(5, 5)
    register_offload_module(disk, "child", child)
    assert isinstance(child._parameters, DiskCache)


def test_align_modules_plain_and_offloaded():
    from compressed_tensors_b200.offload import align_modules

    plain = torch.nn.Linear(1, 1, device=DEV)
    off = _linear()
    offload_module(off, DEV, "cpu")
    with align_modules((plain, off), torch.device("cpu")):
        assert plain.weight.device.type == "cpu" and off.weight.device.type == "cpu"
    assert plain.weight.device == DEV and off.weight.device == DEV


def test_module_forward_call_signature_and_set_item():
    import inspect

    lin = _linear()
    sig = inspect.signature(lin.forward)

    def forward(self, input):
        assert input.device == DEV
        return torch.nn.functional.linear(input, self.weight, self.bias)

    lin.forward = forward.__get__(lin)
    offload_module(lin, DEV, "cpu")
    assert inspect.signature(lin.forward) == inspect.signature(forward.__get__(lin))
    with torch.no_grad():
        assert lin(torch.zeros(5)).device == DEV
    plain = _linear()
    offload_module(plain, DEV, "cpu")
    assert inspect.signature(plain.forward) == sig
    update = torch.nn.Parameter(torch.rand(5, 5), requires_grad=False)
    plain.weight = update   # same shape: written into the existing pinned tensor
    with disable_onloading():
        assert plain.weight is not update and torch.equal(plain.weight, update)
    overwrite = torch.nn.Parameter(torch.rand(6, 6), requires_grad=False)
    plain.weight = overwrite   # new shape: a new pinned copy (the reference keeps the pageable tensor itself)
    with disable_onloading():
        assert plain.weight.is_pinned() and torch.equal(plain.weight, overwrite)
    for size in (5, 6):
        new = torch.rand(size)
        plain.register_buffer("buffer", new, persistent=False)
        with disable_onloading():
            assert torch.equal(plain.buffer, new)


@pytest.mark.parametrize("requires_grad", [True, False])
@pytest.mark.parametrize("device", ["cpu", "cuda:0"])
def test_register_parameter_on_offloaded_module(requires_grad, device):
    lin = _linear()
    offload_module(lin, DEV, "cpu")
    param = torch.nn.Parameter(torch.ones(5, device=device), requires_grad=requires_grad)
    lin.register_parameter("param_name", param)
    assert lin.param_name.device == DEV and torch.equal(lin.param_name.to(device), param)
    with disable_offloading():
        kept = lin.weight
        assert kept in set(OffloadCache.keep_onloaded_values.values())
        new = torch.nn.Parameter(torch.ones(5, 5, device=device), requires_grad=requires_grad)
        lin.weight = new
        assert lin.weight.device == DEV and torch.equal(lin.weight, new.to(DEV))


# ---- review follow-ups: ties, trainability, lifecycle on offloaded models, bounded host queues ------------------------------------
def test_tied_weights_stay_tied_and_trainable():
    from transformers import LlamaConfig, LlamaForCausalLM

    torch.manual_seed(0)
    model = LlamaForCausalLM(LlamaConfig(num_hidden_layers=1, hidden_size=64, num_attention_heads=2, num_key_value_heads=1,
                                         head_dim=32, vocab_size=128, intermediate_size=128, tie_word_embeddings=True))
    assert model.lm_head.weight is model.model.embed_tokens.weight
    set_onload_device(model, DEV)
    with disable_onloading():
        emb, head = model.model.embed_tokens.weight, model.lm_head.weight
        assert emb is head and emb.is_pinned() and emb.requires_grad
    update_offload_parameter(model.model.embed_tokens, "weight", torch.zeros(128, 64))
    assert torch.equal(model.lm_head.weight.cpu(), torch.zeros(128, 64))
    remove_dispatch(model)
    assert model.lm_head.weight.requires_grad and model.lm_head.weight is model.model.embed_tokens.weight


def test_apply_quantization_config_on_offloaded_model():
    from compressed_tensors_b200.quantization import QuantizationConfig, apply_quantization_config
    from compressed_tensors_b200.quantization.utils import calculate_qparams

    torch.manual_seed(3)
    model = torch.nn.Sequential(torch.nn.Linear(256, 128, bias=False), torch.nn.Linear(128, 256, bias=False)).to(BF)
    on_gpu = copy.deepcopy(model).to(DEV)
    set_onload_device(model, DEV)
    for m in (on_gpu, model):
        apply_quantization_config(m, QuantizationConfig(config_groups={"W4A16": ["Linear"]}))
    for a, b in zip(on_gpu, model):
        assert isinstance(b._parameters, CPUCache)
        with disable_onloading():
            assert b._parameters["weight_scale"].device.type == "cpu"
        args = a.quantization_scheme.weights
        w = a.weight.detach().unflatten(-1, (-1, args.group_size))
        s, z = calculate_qparams(w.amin(-1), w.amax(-1), args)
        for m in (a, b):
            update_offload_parameter(m, "weight_scale", s.to(a.weight_scale.dtype))
            if hasattr(a, "weight_zero_point"):
                update_offload_parameter(m, "weight_zero_point", z.to(a.weight_zero_point.dtype))
    x = torch.randn(4, 256, dtype=BF)
    with torch.no_grad():
        want = on_gpu(x.to(DEV))
        got = model(x)   # a CPU input: the offload wrapper moves it before the quantized forward
    assert got.device == DEV and torch.equal(got, want)


@pytest.mark.parametrize("kind", ["cpu", "disk"])
def test_host_queue_split_by_budget_and_pin_failure_are_bit_identical(kind, tmp_path, monkeypatch):
    from compressed_tensors_b200.compressors import ModelCompressor
    from compressed_tensors_b200.compressors.model_compressors import batched

    model = _quantized_model("W4A16")
    on_gpu = copy.deepcopy(model).to(DEV)
    for m in model:
        offload_module(m, DEV, kind, **({"offload_dir": str(tmp_path)} if kind == "disk" else {}))
    mc = ModelCompressor.from_pretrained_model(on_gpu)
    calls = []
    real = ops.host_batched
    monkeypatch.setattr(ops, "host_batched", lambda op, probs, *a: (calls.append(len(probs)), real(op, probs, *a))[1])
    monkeypatch.setattr(batched, "_host_budget", lambda: 1 << 20)   # each 1-3 MiB weight is a part of its own

    def no_pin(shape, dtype):
        raise RuntimeError("pinning refused")

    monkeypatch.setattr(batched, "_pinned_empty", no_pin)
    def offloaded_bytes():
        got = {}
        for i, m in enumerate(model):
            cache = m._parameters
            for k, v in cache.offloaded_values.items():
                if v is not None:
                    got[f"{i}.{k}"] = cache.read(v, "cpu") if kind == "disk" else v
        return got

    mc.compress_model(on_gpu)
    mc.compress_model(model)
    assert calls == [1, 1, 1], calls
    _same_bytes(offloaded_bytes(), {f"{i}.{k}": v for i, m in enumerate(on_gpu) for k, v in m.state_dict().items()},
                f"{kind} split queue, pageable outputs, compressed")
    mc.decompress_model(on_gpu)
    mc.decompress_model(model)
    assert calls == [1, 1, 1, 1, 1, 1], calls
    _same_bytes(offloaded_bytes(), {f"{i}.{k}": v for i, m in enumerate(on_gpu) for k, v in m.state_dict().items()},
                f"{kind} split queue, pageable outputs, decompressed")
