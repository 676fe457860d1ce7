"""Launch variants the default plans do not reach on the suite's usual shapes, each checked element-wise against fp64
(tests/gpu_reference.py: standalone rotate kernel + fp64 matmul on the kernel's own dequantised operand, bias in T):

  * krot != 8 through every fused path the default dispatch takes: decode with in-kernel rotation (the runtime krot loop)
    and with the rotation pre-pass (its masked / second chunk of 8 rotations), the stream kernel, a chain whose steps differ
    in krot and group size, and the GEMM; plus the CPU oracle normwise, so a bug shared by the rotate kernel and the fused
    kernels cannot hide;
  * every GEMM token tile (32, 64, 128) with a ragged last tile, over 1, 2, 9 and 112 rounds of K;
  * forced plans, one child process each (the planner knobs are read once per process): every decode cluster size, the
    fall-back from decode to the stream kernel, the stream kernel at 3 and 16 K slices, in-kernel rotation up to M = 16 and
    the pre-pass from M = 2, the GEMM for M <= 16, and the shallowest weight ring.  Every variant also runs a selection-weight
    layer (tests/selection_layers.py), whose output must equal its exact products element for element.  The parent asserts
    the plan the child logged (PARO_DECODE_VERBOSE=1) and the number of launches, not only the numbers.
"""
import ctypes
import json
import os
import re
import subprocess
import sys
from collections import defaultdict
from pathlib import Path

import pytest
import torch

from gpu_reference import check, check_linear, rotated
from paroquant_b200 import _cabi
from paroquant_b200.checkpoint import make_synthetic_activations, make_synthetic_layer

HERE = Path(__file__).resolve().parent
_TD = {"float16": torch.float16, "bfloat16": torch.bfloat16}
KROTS = [1, 2, 3, 7, 8, 9, 16]          # 8: the unrolled path, as the control


def _report(area, ratio):
    print(f"[max err/tol] {area}: {ratio:.3f}")


@pytest.fixture(scope="module")
def mods():
    import paroquant_b200.kernels.cuda  # noqa: F401  registers torch.ops.rotation.rotate
    from paroquant_b200 import chain
    from paroquant_b200.linear import ParoLinearKernel
    return chain, ParoLinearKernel


def _one_step_chain(chain, k, x, bias, M):
    y = torch.empty(M, k.shape.out_features, dtype=x.dtype, device="cuda")
    chain.ParoChain([chain.ChainStep(k, x=x, y=y, bias=bias)], M)()
    return y


# ---------------------------------------------------------------- krot != 8, default dispatch
@pytest.mark.gpu
@pytest.mark.parametrize("group,dt", [(128, "bfloat16"), (64, "float16")])
@pytest.mark.parametrize("krot", KROTS)
def test_krot_every_fused_path(mods, krot, group, dt):
    """decode in-kernel rotation (M = 1, 2, 4), decode after the pre-pass (M = 5, 16), GEMM (M = 33, 300) through the single
    linear; the stream kernel as a one-step chain (M = 1, 4, 16)."""
    chain, PK = mods
    T = _TD[dt]
    worst = 0.0
    for K, parts, with_bias in ((1024, [256, 128], True), (2048, [384], False)):
        L = make_synthetic_layer(K, parts, group_size=group, krot=krot, seed=400 + krot, device="cuda", bias=with_bias)
        k = PK.from_buffers(L, T, max_m=300)
        W = k.dense_weight()
        bias = None if L.bias is None else L.bias.to(T)
        for M in (1, 2, 4, 5, 16, 33, 300):
            x = make_synthetic_activations(M, K, seed=410 + M, device="cuda", dtype=T)
            y = k(x, bias)
            assert _cabi.last_launch_count() == (1 if M < 5 else 2), M      # in-kernel rotation below 5 rows, a pre-pass from 5
            worst = max(worst, check(y, rotated(L, x), W, parts, bias, what=f"K={K} {parts} M={M}"))
            assert torch.equal(k(x, bias), y)
        for M in (1, 4, 16):
            x = make_synthetic_activations(M, K, seed=420 + M, device="cuda", dtype=T)
            y = _one_step_chain(chain, k, x, bias, M)
            worst = max(worst, check(y, rotated(L, x), W, parts, bias, what=f"stream K={K} {parts} M={M}"))
            assert torch.equal(_one_step_chain(chain, k, x, bias, M), y)
    _report(f"krot {krot} g{group} {dt}", worst)


@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 5, 16])
def test_chain_steps_with_different_krot_and_group(mods, M):
    """Three chained steps with krot 3 / 16 / 9 and group 64 / 128 / 64: the metadata size and the record (ring stage) size
    differ per step.  Each step against the reference on the GPU's own previous output."""
    chain, PK = mods
    T = torch.bfloat16
    specs = [(512, [768], 64, 3), (768, [256, 128], 128, 16), (384, [512], 64, 9)]
    Ls = [make_synthetic_layer(K, parts, group_size=g, krot=r, seed=430 + i, device="cuda") for i, (K, parts, g, r) in enumerate(specs)]
    ks = [PK.from_buffers(L, T) for L in Ls]
    x = make_synthetic_activations(M, 512, seed=440 + M, device="cuda", dtype=T)
    ys = [torch.empty(M, sum(p), dtype=T, device="cuda") for _, p, _, _ in specs]
    ch = chain.ParoChain([chain.ChainStep(ks[0], x=x, y=ys[0]), chain.ChainStep(ks[1], y=ys[1]), chain.ChainStep(ks[2], y=ys[2])], M)
    ch()
    first = [y.clone() for y in ys]
    worst = 0.0
    for i, (L, k, y) in enumerate(zip(Ls, ks, ys)):
        worst = max(worst, check_linear(k, L, x if i == 0 else ys[i - 1], y, what=f"step {i}"))
    ch()
    assert all(torch.equal(a, b) for a, b in zip(ys, first))
    _report(f"3-step chain M={M}", worst)


@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 300])
def test_krot16_llama_qkv(mods, M):
    chain, PK = mods
    L = make_synthetic_layer(4096, [4096, 1024, 1024], krot=16, seed=450, device="cuda")
    k = PK.from_buffers(L, torch.bfloat16, max_m=M)
    x = make_synthetic_activations(M, 4096, seed=451, device="cuda")
    y = k(x)
    _report(f"krot 16 Llama qkv M={M}", check_linear(k, L, x, y, what=f"M={M}"))
    assert torch.equal(k(x), y)


@pytest.mark.gpu
@pytest.mark.parametrize("krot", [1, 2, 3, 7, 9, 16])
def test_krot_vs_oracle(mods, oracle, krot):
    """Independent of the rotate kernel: the CPU oracle (correctly rounded sin / cos), normwise < 1e-3."""
    chain, PK = mods
    L = make_synthetic_layer(1024, [256, 128], krot=krot, seed=460 + krot)
    k = PK.from_buffers(L.to("cuda"), torch.bfloat16)
    cache = {}
    for M in (1, 5, 33):
        x = make_synthetic_activations(M, 1024, seed=470 + M)
        y = k(x.cuda()).float().cpu().numpy()
        ref = oracle.linear(x.float().numpy(), L.numpy_dict(), "bfloat16", W_cache=cache)
        assert oracle.rel_err(y, ref) < 1e-3, (krot, M)
        if M <= 16:
            ys = _one_step_chain(chain, k, x.cuda(), None, M).float().cpu().numpy()
            assert oracle.rel_err(ys, ref) < 1e-3, (krot, M, "stream kernel")


# ---------------------------------------------------------------- GEMM token tiles
# (K, parts, M, NT, group, dtype, bias): M = q * NT + r with r in {1, NT - 1}; K = 128 / 256 / 1152 / 14336 is 1 / 2 / 9 / 112
# rounds; [272, 16] ends both partitions in a partial 128-column block
GEMM_CASES = [
    (128, [272, 16], 65, 32, 128, "bfloat16", True),
    (128, [272, 16], 95, 32, 64, "float16", False),
    (256, [272, 16], 31, 32, 128, "float16", True),
    (14336, [272, 16], 31, 32, 128, "bfloat16", False),
    (256, [272, 16], 65, 64, 64, "bfloat16", False),
    (1152, [256, 128], 127, 64, 128, "float16", True),
    (14336, [640], 129, 64, 128, "bfloat16", False),
    (128, [4096], 129, 128, 64, "bfloat16", True),
    (256, [272, 16], 4095, 128, 128, "bfloat16", False),
    (1152, [4096, 1024, 1024], 383, 128, 64, "float16", True),
    (14336, [4096], 257, 128, 128, "bfloat16", False),
]


def _gemm_plan(K, parts, M, sms, group=128):
    shape = _cabi.make_shape(K, parts, group, 8, torch.bfloat16)
    out = (ctypes.c_int32 * 2)()
    rc = _cabi.lib().paro_debug_gemm_plan(ctypes.byref(shape), M, sms, out)
    if rc:
        raise RuntimeError(_cabi.lib().paro_last_error().decode())
    return tuple(out)


def test_gemm_tile_plan():
    """The tile each GEMM case relies on, on a 132-SM H100; M <= 16 (PARO_SMALL_M_MAX=0) always gets NT = 32."""
    for K, parts, M, nt, group, _, _ in GEMM_CASES:
        assert _gemm_plan(K, parts, M, 132, group) == (nt, (M + nt - 1) // nt), (K, parts, M)
    for M in range(1, 17):
        assert _gemm_plan(1024, [256, 128], M, 132)[0] == 32
        assert _gemm_plan(4096, [4096], M, 132)[0] == 32
    assert {_gemm_plan(4096, [4096], 4096, s)[0] for s in (1, 132)} == {128}
    with pytest.raises(RuntimeError, match="bad M"):
        _gemm_plan(1024, [256], 0, 132)


@pytest.mark.gpu
@pytest.mark.parametrize("K,parts,M,nt,group,dt,with_bias", GEMM_CASES)
def test_gemm_tiles(mods, K, parts, M, nt, group, dt, with_bias):
    chain, PK = mods
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert _gemm_plan(K, parts, M, sms, group)[0] == nt, f"this device ({sms} SMs) picks another tile"
    T = _TD[dt]
    L = make_synthetic_layer(K, parts, group_size=group, seed=480 + M, device="cuda", bias=with_bias)
    k = PK.from_buffers(L, T, max_m=M)
    bias = None if L.bias is None else L.bias.to(T)
    x = make_synthetic_activations(M, K, seed=490 + M, device="cuda", dtype=T)
    y = k(x, bias)
    assert _cabi.last_launch_count() == 2
    _report(f"GEMM NT={nt} K={K} M={M}", check_linear(k, L, x, y, bias, what=f"NT={nt}"))
    assert torch.equal(k(x, bias), y)


# ---------------------------------------------------------------- forced plans, one child process each
_KNOBS = ("PARO_DECODE_C", "PARO_NO_CLUSTER", "PARO_DECODE_STREAM", "PARO_DECODE_PREROT_M", "PARO_SMALL_M_MAX", "PARO_DECODE_STAGES",
          "PARO_DECODE_INFLIGHT", "PARO_DECODE_B8", "PARO_DECODE_VERBOSE")
VARIANTS = {
    "decode_c1": {"PARO_DECODE_C": "1"},
    "decode_c2": {"PARO_DECODE_C": "2"},
    "decode_c4": {"PARO_DECODE_C": "4"},
    "decode_c8": {"PARO_DECODE_C": "8"},
    "stream_c3": {"PARO_DECODE_C": "3"},
    "stream_c16": {"PARO_DECODE_C": "16"},
    "no_cluster": {"PARO_NO_CLUSTER": "1"},
    "stream_only": {"PARO_DECODE_STREAM": "1"},
    "prerot_never": {"PARO_DECODE_PREROT_M": "1"},
    "prerot_from2": {"PARO_DECODE_PREROT_M": "2"},
    "gemm_only": {"PARO_SMALL_M_MAX": "0"},
    "shallow_ring": {"PARO_DECODE_STAGES": "4", "PARO_DECODE_INFLIGHT": "1", "PARO_DECODE_B8": "0"},
}


def _observed(stderr):
    """Launch plans the library logged, per case: decode cluster sizes and stages, stream K slices, stages and B rows."""
    obs, cur = {}, None
    for line in stderr.splitlines():
        if line.startswith("[case] "):
            cur = obs.setdefault(line[7:], defaultdict(set))
        elif cur is not None and (m := re.search(r"\[paro decode\] .*: cluster (\d+) x .*, (\d+) stages", line)):
            cur["decode"].add(int(m[1]))
            cur["dec_stages"].add(int(m[2]))
        elif cur is not None and (m := re.search(r"\[paro stream\] step \d+ .*: (\d+) slices x", line)):
            cur["stream"].add(int(m[1]))
        elif cur is not None and (m := re.search(r"\[paro stream\] \d+ CTAs, (\d+) stages, B rows (\d+)", line)):
            cur["stm_stages"].add(int(m[1]))
            cur["b_rows"].add(int(m[2]))
    return obs


def _expect(variant, case, o):
    """The plan `variant` must have produced for `case` (its JSON record) given the observations o."""
    M, K, kind, n = case["M"], case["K"], case["kind"], case.get("launches")
    prerot = M >= 5                                 # default rule for K < 8192 (fewer than 64 groups)
    if variant.startswith("decode_c"):
        c = int(variant[len("decode_c"):])
        assert o["decode"] == {c} and not o["stream"], o
        assert n == (2 if prerot else 1)
    elif variant.startswith("stream_c"):
        c = int(variant[len("stream_c"):])
        assert not o["decode"] and o["stream"] == {c}, o
        assert kind == "tail" or n == 1                # no pre-pass is launched for a decode plan that does not exist
    elif variant == "no_cluster":
        if K >= 14336:
            assert not o["decode"] and o["stream"], o
            assert n == 1
        else:
            assert o["decode"] == {1} and not o["stream"], o
            assert n == (2 if prerot else 1)
    elif variant == "stream_only":
        assert not o["decode"] and o["stream"] and n == 1, o
    elif variant == "prerot_never":
        assert o["decode"] and not o["stream"] and n == 1, o
    elif variant == "prerot_from2":
        assert o["decode"] and not o["stream"] and n == (2 if M >= 2 else 1), o
    elif variant == "gemm_only":
        assert not o["decode"] and not o["stream"] and n == 2, o
    elif variant == "shallow_ring":
        if kind == "chain1":
            assert not o["decode"] and o["stm_stages"] == {4} and o["b_rows"] == {16}, o
        else:
            assert o["dec_stages"] == {4} and not o["stream"], o
    else:
        raise KeyError(variant)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_forced_variant(variant):
    env = {k: v for k, v in os.environ.items() if k not in _KNOBS}
    env.update(VARIANTS[variant], PARO_DECODE_VERBOSE="1")
    r = subprocess.run([sys.executable, str(HERE / "variant_child.py"), variant], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, f"child exited {r.returncode}\n{r.stderr[-4000:]}"
    summary = json.loads(r.stdout.strip().splitlines()[-1])
    obs = _observed(r.stderr)
    failed = [c for c in summary["cases"] if not c["ok"]]
    assert not failed, "\n".join(f"{c['name']}: {c.get('error')}" for c in failed)
    for case in summary["cases"]:
        o = obs[case["name"]]
        _expect(variant, case, o)
        plan = ", ".join(f"{k}={sorted(v)}" for k, v in sorted(o.items()) if v)
        extra = ("selection weights: every element exact" if case.get("exact") else
                 f"max err/tol {case['ratio']:.3f}" if "ratio" in case else f"stage errors {case['stage_err']}")
        print(f"[plan] {variant}: {case['name']}: {plan}, launches {case.get('launches')}, {extra}")
