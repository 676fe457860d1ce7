"""GPU parity of the fused path (prepack + rotate + dequant + GEMM), through the C-ABI.

  * prepack is integer work: the dense operand read back from the packed layout must equal the
    oracle's T((q - z) * s) BIT FOR BIT;
  * fused linear vs the oracle on the same seeded inputs: normwise relative error <= 1e-3 in the
    activation dtype (BASELINE.json's tolerance); in practice ~1e-4 (MUFU flips in the rotation
    + fp32 accumulation order);
  * vs fixtures of the unmodified reference pipeline (its rotate + vLLM Marlin) captured on an H100;
  * size-independent properties at BASELINE sizes.
"""
import numpy as np
import pytest
import torch

from paroquant_b200.checkpoint import make_synthetic_activations, make_synthetic_layer

from conftest import GOLDEN
from gpu_reference import check_linear

pytestmark = pytest.mark.gpu
TOL = 1e-3
_TD = {"float16": torch.float16, "bfloat16": torch.bfloat16}


@pytest.fixture(scope="module")
def PK():
    from paroquant_b200.linear import ParoLinearKernel
    return ParoLinearKernel


def _oracle_linear(oracle, L, x, dt, cache):
    return oracle.linear(x.float().cpu().numpy(), L.numpy_dict(), dt, W_cache=cache)


@pytest.mark.parametrize("dt", ["bfloat16", "float16"])
@pytest.mark.parametrize("K,parts", [(512, [64]), (1024, [256, 128]), (640, [48, 16, 32]), (4096, [4096])])
def test_prepack_preserves_operand_bit_exact(PK, oracle, dt, K, parts):
    L = make_synthetic_layer(K, parts, seed=41)
    k = PK.from_buffers(L.to("cuda"), _TD[dt])
    W = k.dense_weight().float().cpu().numpy()
    d = L.numpy_dict()
    ref = oracle.c_dequant(d["qweight"], d["qzeros"], d["scales"], 128, dt)
    assert np.array_equal(W, ref)


@pytest.mark.parametrize("dt", ["bfloat16", "float16"])
@pytest.mark.parametrize("K,parts,Ms", [
    (512, [64], (1, 2, 3, 8, 9, 16)),                 # one partial 128-column block
    (1024, [256, 128], (1, 4, 7, 16)),                # merged, different rotation per partition
    (640, [48, 16, 32], (1, 5, 16)),                  # every partition is a partial block, 5 groups over the cluster's K slices
    (256, [272, 16], (3, 12)),                        # two full blocks + a partial one; 12 rows = three rotation row blocks
    (4096, [4096], (1, 4, 16)),                       # BASELINE config 0/1 shape
])
def test_fused_linear_vs_oracle(PK, oracle, dt, K, parts, Ms):
    L = make_synthetic_layer(K, parts, seed=43, bias=(K == 1024))
    k = PK.from_buffers(L.to("cuda"), _TD[dt])
    cache = {}
    bias = None if L.bias is None else L.bias.to("cuda", _TD[dt])
    for M in Ms:
        x = make_synthetic_activations(M, K, seed=50 + M, dtype=_TD[dt])
        y = k(x.cuda(), bias)
        assert y.shape == (M, sum(parts)) and y.dtype == _TD[dt]
        ref = _oracle_linear(oracle, L, x, dt, cache)
        err = oracle.rel_err(y.float().cpu().numpy(), ref)
        assert err < TOL, (M, err)
        # determinism: split-K partials are added in a fixed order
        assert torch.equal(k(x.cuda(), bias), y)


@pytest.mark.parametrize("K,parts", [(4096, [4096, 1024, 1024]), (4096, [14336, 14336]), (14336, [4096]), (11008, [4096])])
def test_llama_shapes_vs_oracle_and_dense(PK, oracle, K, parts):
    """Llama-3-8B merged qkv / gate_up / down (+ Llama-2 K=11008 ragged slices) at M = 1 and 16:
    column samples against the oracle, every element against an fp64 matmul on the kernel's own
    dequantised operand and the standalone rotate kernel (tests/gpu_reference.py)."""
    L = make_synthetic_layer(K, parts, seed=47, device="cuda")
    k = PK.from_buffers(L, torch.bfloat16)
    W = k.dense_weight()
    for M in (1, 16):
        x = make_synthetic_activations(M, K, seed=60 + M, device="cuda")
        check_linear(k, L, x, k(x), W=W, what=f"M={M}")
    # oracle on a column sample (full oracle GEMM at these sizes would take minutes)
    cols = torch.arange(0, sum(parts), max(1, sum(parts) // 257))[:256]
    d = L.to("cpu").numpy_dict()
    x = make_synthetic_activations(1, K, seed=61, device="cuda")
    y = k(x).float().cpu().numpy()[0, cols.numpy()]
    Wc = oracle.c_dequant(d["qweight"], d["qzeros"], d["scales"], 128, "bfloat16")[:, cols.numpy()]
    bounds = np.cumsum([0] + list(parts))
    acc = np.zeros(len(cols))
    for p in range(len(parts)):
        xr = oracle.c_rotate(x.float().cpu().numpy(), d["pairs"][p], d["theta"][p], d["channel_scales"][p], 128, "bfloat16")
        sel = (cols.numpy() >= bounds[p]) & (cols.numpy() < bounds[p + 1])
        acc[sel] = (xr.astype(np.float64) @ Wc[:, sel].astype(np.float64))[0]
    assert oracle.rel_err(y, oracle.round_to(acc.astype(np.float32), "bfloat16")) < TOL


def test_properties_at_full_size(PK):
    """theta = 0 & unit channel scales: the fused kernel must equal x @ dequant(W) with NO rotation;
    linearity in x for power-of-two factors; row independence (batch rows do not interact)."""
    L = make_synthetic_layer(4096, [4096], seed=71, device="cuda")
    L.theta.zero_()
    L.channel_scales.fill_(1.0)
    k = PK.from_buffers(L, torch.bfloat16)
    W = k.dense_weight().double()
    x = make_synthetic_activations(16, 4096, seed=9, device="cuda")
    y = k(x)
    ref = (x.double() @ W).float().to(torch.bfloat16).double()
    assert ((y.double() - ref).norm() / ref.norm()).item() < 3e-4           # identical up to rare one-ulp flips
    assert torch.equal(k(x * 4), y * 4)
    # rows do not interact: replacing the other rows leaves a row's bits unchanged (same M, same summation order) ...
    x2 = torch.randn_like(x)
    for m in (0, 7, 15):
        x2[m] = x[m]
    y2 = k(x2)
    for m in (0, 7, 15):
        assert torch.equal(y2[m], y[m])
    # ... and a different batch size (a different split of K, i.e. another fp32 summation order) moves a row by rounding only
    for xs, ys in ((x[3:4], y[3:4]), (x[:8], y[:8])):
        assert ((k(xs).double() - ys.double()).norm() / ys.double().norm()).item() < 3e-4
    assert torch.equal(k(x), y)   # run to run bit-reproducible


def test_module_surfaces(PK, oracle):
    """RotateQuantizedLinear (HF surface) filled through its state dict, fp16 and bf16; leading
    batch dims; bias."""
    from paroquant_b200.inference.backends.transformers import RotateQuantizedLinear

    L = make_synthetic_layer(1024, [256], seed=81, bias=True)
    m = RotateQuantizedLinear(1024, 256, bias=True)
    m.load_state_dict({"theta": L.theta[0], "pairs": L.pairs[0], "channel_scales": L.channel_scales[0],
                       "qweight": L.qweight, "qzeros": L.qzeros, "scales": L.scales, "bias": L.bias})
    m = m.cuda()
    for dt in ("float16", "bfloat16"):
        x = make_synthetic_activations(6, 1024, seed=3, dtype=_TD[dt]).view(2, 3, 1024)
        y = m(x.cuda())
        assert y.shape == (2, 3, 256)
        ref = oracle.linear(x.float().numpy().reshape(6, 1024), L.numpy_dict(), dt)
        assert oracle.rel_err(y.float().cpu().numpy().reshape(6, 256), ref) < TOL


def test_vllm_linear_method_end_to_end(PK, oracle, monkeypatch):
    """create_weights -> loaders -> process_weights_after_loading -> apply on a bare module."""
    P = pytest.importorskip("paroquant_b200.inference.backends.vllm.plugin")
    import vllm.model_executor.parameter as vp
    monkeypatch.setattr(vp, "get_tensor_model_parallel_rank", lambda: 0)
    monkeypatch.setattr(vp, "get_tensor_model_parallel_world_size", lambda: 1)
    L = make_synthetic_layer(1024, [512, 128, 128], seed=91)
    method = P.ParoQuantLinearMethod(P.ParoQuantConfig(4, 128, 8, True))
    layer = torch.nn.Module()
    method.create_weights(layer, 1024, [512, 128, 128], 1024, 768, torch.bfloat16, weight_loader=None)
    layer.qweight.data.copy_(L.qweight)
    layer.qzeros.data.copy_(L.qzeros)
    layer.scales.data.copy_(L.scales)
    for p, sid in enumerate(("q", "k", "v")):
        P._rotation_weight_loader(layer.theta, L.theta[p], sid)
        P._rotation_weight_loader(layer.pairs, L.pairs[p], sid)
        P._rotation_weight_loader(layer.channel_scales, L.channel_scales[p], sid)
    layer = layer.cuda()
    method.process_weights_after_loading(layer)
    assert not hasattr(layer, "qweight") and layer.rot_theta.shape == (3, 8, 512)
    x = make_synthetic_activations(4, 1024, seed=4)
    y = method.apply(layer, x.cuda(), None)
    ref = oracle.linear(x.float().numpy(), L.numpy_dict(), "bfloat16")
    assert oracle.rel_err(y.float().cpu().numpy(), ref) < TOL


_lin_golden = sorted(GOLDEN.glob("ref_gpu_linear_*.npz"))


@pytest.mark.skipif(not _lin_golden, reason="reference GPU fixtures not generated yet")
@pytest.mark.parametrize("path", _lin_golden, ids=lambda p: p.stem)
def test_vs_reference_pipeline_fixture(PK, path):
    """Same packed weights / scales / rotations as the reference's rotate + Marlin run: outputs
    within 1e-3 (north_star), and the dequantised operand identical to Marlin's, bit for bit."""
    z = np.load(path)
    dt = str(z["dtype"])
    f16 = lambda a: torch.from_numpy(np.ascontiguousarray(a)).view(torch.int16).view(torch.float16)
    k = PK.from_tensors(torch.from_numpy(z["qweight"]).cuda(), torch.from_numpy(z["qzeros"]).cuda(), f16(z["scales"]).cuda(),
                        f16(z["theta"]).cuda(), torch.from_numpy(z["pairs"]).cuda(), f16(z["channel_scales"]).cuda(),
                        [int(v) for v in z["part_sizes"]], dtype=_TD[dt])
    x = torch.from_numpy(np.ascontiguousarray(z["x"])).view(torch.int16).view(_TD[dt]).cuda()
    y = k(x).float().cpu()
    ref = torch.from_numpy(np.ascontiguousarray(z["y"])).view(torch.int16).view(_TD[dt]).float()
    assert ((y - ref).norm() / ref.norm()).item() < TOL
    W = k.dense_weight().cpu()
    wref = torch.from_numpy(np.ascontiguousarray(z["w_onehot"])).view(torch.int16).view(_TD[dt])
    assert torch.equal(W[torch.from_numpy(z["w_rows"])], wref)


@pytest.mark.parametrize("dt", ["bfloat16", "float16"])
@pytest.mark.parametrize("K,parts,M", [(512, [128], 17), (1024, [256, 128], 40), (1024, [256, 128], 64), (4096, [1024], 100),
                                       (4096, [4096], 256), (4096, [4096, 1024, 1024], 300), (11008, [512], 33), (14336, [256], 257),
                                       (1152, [128], 40), (256, [272, 16], 33)])
def test_large_m_gemm_vs_rotate_and_dense(PK, dt, K, parts, M):
    """M > 16: rotation pre-pass + wgmma GEMM, every element against an fp64 matmul on the kernel's own dequantised operand
    and the standalone rotate kernel (both bit-checked elsewhere; tests/gpu_reference.py); ragged M (not a multiple of the
    token tile), merged projections, K longer than the weight ring (stage reuse), partial 128-column blocks."""
    L = make_synthetic_layer(K, parts, seed=53, device="cuda", bias=(M == 40))
    k = PK.from_buffers(L, _TD[dt], max_m=M)
    x = make_synthetic_activations(M, K, seed=70 + M, device="cuda", dtype=_TD[dt])
    bias = None if L.bias is None else L.bias.to(_TD[dt])
    y = k(x, bias)
    check_linear(k, L, x, y, bias, what=f"M={M}")
    assert torch.equal(k(x, bias), y)


def test_large_m_vs_oracle(PK, oracle):
    L = make_synthetic_layer(1024, [256, 128], seed=59)
    k = PK.from_buffers(L.to("cuda"), torch.bfloat16, max_m=48)
    x = make_synthetic_activations(48, 1024, seed=12)
    y = k(x.cuda()).float().cpu().numpy()
    ref = oracle.linear(x.float().numpy(), L.numpy_dict(), "bfloat16")
    assert oracle.rel_err(y, ref) < TOL


@pytest.mark.parametrize("name,K,parts", [("qkv", 4096, [4096, 1024, 1024]), ("o", 4096, [4096]), ("gate_up", 4096, [14336, 14336]),
                                          ("down", 14336, [4096]), ("llama2_down", 11008, [4096])])
def test_prefill_4096_vs_oracle_samples(PK, oracle, name, K, parts):
    """The batch bench.py's `prefill` section reports (4096 tokens, Llama-3-8B shapes, plus K = 11008): sampled token rows
    x sampled output columns against the oracle (its rotate on the sampled rows, its dequant on the sampled columns, its
    fp32 GEMM), every partition and the last partial token tile included."""
    M = 4096
    L = make_synthetic_layer(K, parts, seed=97)
    k = PK.from_buffers(L.to("cuda"), torch.bfloat16, check_pairs=False, max_m=M)
    x = make_synthetic_activations(M, K, seed=98)
    y = k(x.cuda()).float().cpu().numpy()
    rows = np.array([0, 1, 255, 256, 1023, 2048, 4095])
    d = L.numpy_dict()
    W = None
    n0 = 0
    for p, n in enumerate(parts):
        cols = n0 + np.array(sorted({0, 1, 127, 128, n // 2 + 5, n - 129, n - 1}))
        xr = oracle.c_rotate(x[rows].float().numpy(), d["pairs"][p], d["theta"][p], d["channel_scales"][p], 128, "bfloat16")
        if W is None:
            W = oracle.c_dequant(d["qweight"], d["qzeros"], d["scales"], 128, "bfloat16")
        ref = oracle.c_gemm(xr, np.ascontiguousarray(W[:, cols]), None, "bfloat16")
        got = y[np.ix_(rows, cols)]
        assert oracle.rel_err(got, ref) < TOL, (name, p)
        n0 += n


def test_linear_op_is_opaque_under_torch_compile(PK):
    """vLLM traces `ParoQuantLinearMethod.apply` with fullgraph=True and a symbolic batch dimension: the call must be ONE opaque
    op (no ctypes, no Python branch on the row count in `ParoLinearKernel.__call__`), for decode and prefill sizes alike."""
    L = make_synthetic_layer(1024, [256, 128], seed=77, bias=True)
    k = PK.from_buffers(L.to("cuda"), torch.bfloat16, check_pairs=False)   # default max_m = 16: prefill sizes must still work
    bias = L.bias.to("cuda")                                                # fp16 checkpoint bias meets bf16 activations

    def f(x):
        return k(x * 1.0, bias) + 0.0

    cf = torch.compile(f, fullgraph=True, dynamic=True)
    for M in (1, 7, 48, 300):
        x = make_synthetic_activations(M, 1024, seed=M, device="cuda")
        assert torch.equal(cf(x), f(x))


# ---------------------------------------------------------------- group_size 64
# The converter rotates AND quantises in groups of `group_size` (cli/convert.py:176-182) and the rotate op dispatches 64 and
# 128 (rotation.cu:117-123).  The reference's inference call sites drop the argument (plugin.py:285, modules.py:59 rotate with
# the default 128), so there is no reference pipeline to compare with: the oracle with group = 64 on both halves is the bar.
@pytest.mark.parametrize("dt", ["bfloat16", "float16"])
@pytest.mark.parametrize("K,parts", [(512, [64]), (1024, [256, 128]), (640, [48, 16, 32])])
def test_group64_prepack_preserves_operand_bit_exact(PK, oracle, dt, K, parts):
    L = make_synthetic_layer(K, parts, group_size=64, seed=141)
    k = PK.from_buffers(L.to("cuda"), _TD[dt])
    d = L.numpy_dict()
    assert np.array_equal(k.dense_weight().float().cpu().numpy(), oracle.c_dequant(d["qweight"], d["qzeros"], d["scales"], 64, dt))


@pytest.mark.parametrize("dt", ["bfloat16", "float16"])
@pytest.mark.parametrize("K,parts,Ms", [
    (512, [64], (1, 2, 5, 16, 17)),                   # cluster kernel, pre-rotated rows from 5 on, GEMM path at 17
    (1024, [256, 128], (1, 4, 16, 48, 300)),          # merged; 48 / 300 rows: rotation pre-pass + wgmma GEMM
    (640, [48, 16, 32], (3, 12)),
    (4096, [4096], (1, 16)),
])
def test_group64_fused_linear_vs_oracle(PK, oracle, dt, K, parts, Ms):
    L = make_synthetic_layer(K, parts, group_size=64, seed=143, bias=(K == 1024))
    assert int(L.numpy_dict()["group"]) == 64
    k = PK.from_buffers(L.to("cuda"), _TD[dt])
    cache = {}
    bias = None if L.bias is None else L.bias.to("cuda", _TD[dt])
    for M in Ms:
        x = make_synthetic_activations(M, K, seed=150 + M, dtype=_TD[dt])
        y = k(x.cuda(), bias)
        ref = _oracle_linear(oracle, L, x, dt, cache)
        err = oracle.rel_err(y.float().cpu().numpy(), ref)
        assert err < TOL, (M, err)
        assert torch.equal(k(x.cuda(), bias), y)


def test_group64_rotation_equals_the_standalone_op(PK):
    """theta as drawn, unit weights are not needed: the fused kernel on a group-64 layer equals the standalone rotate op run
    with group_size = 64 followed by a matmul on the kernel's own dequantised operand."""
    import paroquant_b200.kernels.cuda  # noqa: F401
    L = make_synthetic_layer(2048, [384], group_size=64, seed=147, device="cuda")
    k = PK.from_buffers(L, torch.bfloat16)
    W = k.dense_weight().double()
    for M in (1, 16, 64):
        x = make_synthetic_activations(M, 2048, seed=160 + M, device="cuda")
        xr = torch.ops.rotation.rotate(x, L.pairs[0], L.theta[0], L.channel_scales[0], 64)
        ref = (xr.double() @ W).float().to(torch.bfloat16).double()
        err = ((k(x).double() - ref).norm() / ref.norm()).item()
        assert err < 3e-4, (M, err)
