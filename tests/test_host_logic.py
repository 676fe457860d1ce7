"""Host-side mirror of the reference surface, on CPU: checkpoint helpers, module / plugin
parameter surfaces, rotation-parameter loaders, TP sharding arithmetic."""
import numpy as np
import pytest
import torch

from paroquant_b200.checkpoint import ParoLayerBuffers, make_synthetic_layer, validate_pairs
from paroquant_b200.parallel import shard_columns, shard_rows


def test_synthetic_layer_is_deterministic_and_valid():
    a = make_synthetic_layer(512, [256, 128], seed=3)
    b = make_synthetic_layer(512, [256, 128], seed=3)
    for f in ("qweight", "qzeros", "scales", "theta", "pairs", "channel_scales"):
        assert torch.equal(getattr(a, f), getattr(b, f))
    assert a.theta.shape == (2, 8, 256) and a.pairs.shape == (2, 8, 512) and a.channel_scales.shape == (2, 1, 512)
    validate_pairs(a.pairs, 128)
    bad = a.pairs.clone()
    bad[0, 0, 0] = bad[0, 0, 1]
    with pytest.raises(ValueError, match="permutation"):
        validate_pairs(bad, 128)


def test_algorithmic_bytes_match_survey_table():
    # SURVEY.md section 8(d): 4096x4096 -> 8,839,168 B at M = 1; merged qkv -> 13,414,400 B
    L = ParoLayerBuffers(torch.zeros(4096, 512, dtype=torch.int32), None, None, torch.zeros(1, 8, 2048), None, None, [4096])
    assert L.algorithmic_bytes(1) == 8_839_168
    L = ParoLayerBuffers(torch.zeros(4096, 768, dtype=torch.int32), None, None, torch.zeros(3, 8, 2048), None, None, [4096, 1024, 1024])
    assert L.algorithmic_bytes(1) == 13_414_400


def test_rotate_quantized_linear_surface():
    from paroquant_b200.inference.backends.transformers import RotateQuantizedLinear

    m = RotateQuantizedLinear(4096, 1024, bias=True)
    sd = m.state_dict()
    assert {k: (tuple(v.shape), v.dtype) for k, v in sd.items()} == {
        "theta": ((8, 2048), torch.float16), "pairs": ((8, 4096), torch.int16),
        "channel_scales": ((1, 4096), torch.float16), "qweight": ((4096, 128), torch.int32),
        "qzeros": ((32, 128), torch.int32), "scales": ((32, 1024), torch.float16), "bias": ((1024,), torch.float16)}
    with pytest.raises(RuntimeError, match="float16 or bfloat16"):
        m(torch.zeros(1, 4096))
    with pytest.raises(RuntimeError, match="CUDA-only"):   # no CPU fallback
        m(torch.zeros(1, 4096, dtype=torch.float16))


def test_row_shards_recompose(oracle):
    """Sum over K-shards of oracle(linear on shard) == oracle(full) before the final rounding:
    rotation groups and quant groups never straddle a 128-aligned K-shard."""
    full = make_synthetic_layer(1024, [64], seed=9)
    x = torch.randn(3, 1024).numpy()
    d = full.numpy_dict()
    xr = oracle.c_rotate(x, d["pairs"][0], d["theta"][0], d["channel_scales"][0], 128, "bfloat16")
    W = oracle.c_dequant(d["qweight"], d["qzeros"], d["scales"], 128, "bfloat16")
    acc_full = xr.astype(np.float64) @ W.astype(np.float64)
    acc = 0
    for r in range(4):
        s = shard_rows(full, r, 4)
        assert s.in_features == 256 and s.theta.shape[-1] == 128 and s.qzeros.shape[0] == 2
        ds = s.numpy_dict()
        xs = x[:, r * 256:(r + 1) * 256]
        xrs = oracle.c_rotate(xs, ds["pairs"][0], ds["theta"][0], ds["channel_scales"][0], 128, "bfloat16")
        assert (xrs == xr[:, r * 256:(r + 1) * 256]).all()
        acc = acc + xrs.astype(np.float64) @ oracle.c_dequant(ds["qweight"], ds["qzeros"], ds["scales"], 128, "bfloat16").astype(np.float64)
    assert np.allclose(acc, acc_full, rtol=1e-12, atol=1e-12)
    with pytest.raises(ValueError, match="group boundaries"):
        shard_rows(make_synthetic_layer(1280, [64]), 0, 4)   # 10 groups, like 11008/8 = 10.75


def test_row_shards_recompose_group64(oracle):
    """group_size 64: rotation and quantisation groups are 64 channels, a shard still has to be a whole number of 128-channel
    weight records; the oracle on the shards adds up to the oracle on the full layer."""
    full = make_synthetic_layer(512, [64], group_size=64, seed=19)
    x = torch.randn(2, 512).numpy()
    d = full.numpy_dict()
    assert d["group"] == 64 and d["qzeros"].shape[0] == 8
    xr = oracle.c_rotate(x, d["pairs"][0], d["theta"][0], d["channel_scales"][0], 64, "float16")
    acc_full = xr.astype(np.float64) @ oracle.c_dequant(d["qweight"], d["qzeros"], d["scales"], 64, "float16").astype(np.float64)
    acc = 0
    for r in range(2):
        s = shard_rows(full, r, 2)
        assert s.in_features == 256 and s.group_size == 64 and s.qzeros.shape[0] == 4
        ds = s.numpy_dict()
        xrs = oracle.c_rotate(x[:, r * 256:(r + 1) * 256], ds["pairs"][0], ds["theta"][0], ds["channel_scales"][0], 64, "float16")
        assert (xrs == xr[:, r * 256:(r + 1) * 256]).all()
        acc = acc + xrs.astype(np.float64) @ oracle.c_dequant(ds["qweight"], ds["qzeros"], ds["scales"], 64, "float16").astype(np.float64)
    assert np.allclose(acc, acc_full, rtol=1e-12, atol=1e-12)
    with pytest.raises(ValueError, match="128-channel group boundaries"):
        shard_rows(make_synthetic_layer(384, [64], group_size=64), 0, 2)   # 192 channels per rank: whole groups, but half a record


def test_column_shards_recompose(oracle):
    full = make_synthetic_layer(256, [64, 32], seed=10, bias=True)
    d = full.numpy_dict()
    W = oracle.c_dequant(d["qweight"], d["qzeros"], d["scales"], 128, "float16")
    cols = []
    for r in range(2):
        s = shard_columns(full, r, 2)
        assert s.part_sizes == [32, 16]
        ds = s.numpy_dict()
        cols.append(oracle.c_dequant(ds["qweight"], ds["qzeros"], ds["scales"], 128, "float16"))
    got = np.concatenate([cols[0][:, :32], cols[1][:, :32], cols[0][:, 32:], cols[1][:, 32:]], axis=1)
    assert (got == W).all()


@pytest.fixture
def vllm_plugin(monkeypatch):
    P = pytest.importorskip("paroquant_b200.inference.backends.vllm.plugin")
    import vllm.model_executor.parameter as vp

    monkeypatch.setattr(vp, "get_tensor_model_parallel_rank", lambda: 0)
    monkeypatch.setattr(vp, "get_tensor_model_parallel_world_size", lambda: 1)
    return P


def test_vllm_plugin_surface(vllm_plugin, monkeypatch):
    P = vllm_plugin
    from vllm.model_executor.layers.quantization import get_quantization_config

    assert get_quantization_config("paroquant") is P.ParoQuantConfig
    cfg = P.ParoQuantConfig.from_config({"quant_method": "paroquant", "bits": 4, "group_size": 128, "krot": 8})
    assert (cfg.bits, cfg.group_size, cfg.krot, cfg.zero_point, cfg.pack_factor) == (4, 128, 8, True, 8)
    assert cfg.get_name() == "paroquant" and cfg.get_min_capability() == 90
    assert cfg.get_supported_act_dtypes() == [torch.half, torch.bfloat16]
    with pytest.raises(ValueError, match="Unsupported bits"):
        P.ParoQuantConfig(3, 128, 8, True)

    method = P.ParoQuantLinearMethod(cfg)
    layer = torch.nn.Module()
    method.create_weights(layer, 4096, [4096, 1024, 1024], 4096, 6144, torch.bfloat16, weight_loader=lambda *a, **k: None)
    shapes = {n: (tuple(p.shape), p.dtype) for n, p in layer.named_parameters()}
    assert shapes == {"qweight": ((4096, 768), torch.int32), "qzeros": ((32, 768), torch.int32),
                      "scales": ((32, 6144), torch.bfloat16), "theta": ((3, 8, 2048), torch.float16),
                      "pairs": ((3, 8, 4096), torch.int16), "channel_scales": ((3, 1, 4096), torch.float16)}
    assert layer.num_partitions == 3 and layer.output_partition_sizes == [4096, 1024, 1024]

    # loaders: shard ids None | "q"/"k"/"v" | int | tuple  (plugin.py:53-76 of the reference)
    th = torch.arange(8 * 2048, dtype=torch.float16).view(8, 2048)
    P._rotation_weight_loader(layer.theta, th, "k")
    assert torch.equal(layer.theta.data[1], th) and layer.theta.data[0].abs().sum() == 0
    P._rotation_weight_loader(layer.theta, th + 1, (0, 2))
    assert torch.equal(layer.theta.data[0], th + 1) and torch.equal(layer.theta.data[2], th + 1)
    one = torch.nn.Module()
    method.create_weights(one, 4096, [4096], 4096, 4096, torch.float16, weight_loader=lambda *a, **k: None)
    P._rotation_weight_loader(one.pairs, torch.ones(8, 4096, dtype=torch.int16), None)
    assert one.pairs.data.sum() == 8 * 4096

    # row-parallel: param allocated for K/tp, checkpoint holds K -> slice by rank
    import vllm.distributed as vd
    monkeypatch.setattr(vd, "get_tensor_model_parallel_rank", lambda: 1)
    half = torch.nn.Module()
    method.create_weights(half, 2048, [4096], 4096, 4096, torch.float16, weight_loader=lambda *a, **k: None)
    full_cs = torch.arange(4096, dtype=torch.float16).view(1, 4096)
    P._rotation_weight_loader(half.channel_scales, full_cs, None)
    assert torch.equal(half.channel_scales.data[0], full_cs[:, 2048:])
    with pytest.raises(ValueError, match="incompatible shapes"):
        P._maybe_shard_input(torch.zeros(1, 3000), full_cs)
    with pytest.raises(ValueError, match="multiples of 16"):
        method.create_weights(torch.nn.Module(), 4096, [100], 4096, 100, torch.float16, weight_loader=None)


def test_vllm_entry_point_is_idempotent(vllm_plugin):
    from paroquant_b200.inference.backends.vllm import register

    register()
    register()
    assert hasattr(torch.ops.rotation, "rotate") and hasattr(torch.ops.paro, "linear")


def test_shared_workspace_grows_without_invalidating_old_buffers():
    """All linears of a device share one scratch buffer (scratch behind a 256-byte head holding the launch epoch); growing
    it is geometric (a batch size that creeps up allocates O(log) buffers) and keeps the previous buffers alive -- CUDA
    graphs captured earlier hold their pointers."""
    import torch
    from paroquant_b200 import linear
    dev = torch.device("cpu")
    linear._shared_scratch.pop(dev, None)
    a = linear.shared_workspace(dev, 10)
    assert a.numel() >= 256 and linear.shared_workspace(dev, 200) is a and int(a.sum()) == 0
    n = a.numel()
    b = linear.shared_workspace(dev, n + 1)
    assert b.numel() >= 2 * n and b is not a and linear.shared_workspace(dev, n) is b
    sizes = {linear.shared_workspace(dev, n + 4096 * i).numel() for i in range(1, 200)}
    assert len(sizes) <= 3, "growth must be geometric"
    assert any(t is a for t in linear._shared_scratch[dev])          # still referenced
