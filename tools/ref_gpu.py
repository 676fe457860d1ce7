"""Run the UNMODIFIED reference pipeline on a GPU: its own rotate kernel (oracle/_ref/
paroquant_rotation.so, built by oracle/build_ref.py from /root/reference) followed by vLLM's
AWQ-Marlin GEMM -- i.e. what ParoQuantLinearMethod.apply executes
(/root/reference/paroquant/inference/backends/vllm/plugin.py:281-311).

Always a separate process: the reference library registers the same `rotation::rotate` op name
as paroquant_b200.kernels.cuda.  Nothing from paroquant_b200's kernels is imported here.

    python tools/ref_gpu.py golden  <outdir>          fixtures for tests/golden/
    python tools/ref_gpu.py samples <out.npz>         seeded samples of the outputs of PIPELINE_CASES (tests/test_gpu_reference.py)
    python tools/ref_gpu.py bench   <out.json> [--m 1,16,4096]  per-linear timings of rotate + Marlin (CUDA graph)
"""
from __future__ import annotations

import json
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from paroquant_b200.checkpoint import make_synthetic_activations, make_synthetic_layer  # noqa: E402

REF_SO = ROOT / "oracle" / "_ref" / "paroquant_rotation.so"
_TD = {"float32": torch.float32, "float16": torch.float16, "bfloat16": torch.bfloat16}


def load_reference_rotate():
    if not REF_SO.exists():
        raise SystemExit(f"{REF_SO} missing: run `python oracle/build_ref.py` where /root/reference exists")
    torch.ops.load_library(str(REF_SO))
    return torch.ops.rotation.rotate


def bits(t: torch.Tensor) -> np.ndarray:
    t = t.detach().cpu().contiguous()
    if t.dtype == torch.float32:
        return t.numpy()
    return t.view(torch.int16).numpy().view(np.uint16)


class MarlinLinear:
    """AWQ buffers of ONE partition repacked for vLLM's Marlin, as plugin.py:208-249 does."""

    def __init__(self, qweight, qzeros, scales, K, N, dtype):
        from vllm import _custom_ops as ops
        from vllm.model_executor.layers.quantization.utils import marlin_utils as mu
        from vllm.scalar_type import scalar_types

        dev = qweight.device
        self.K, self.N = K, N
        self.qw = ops.awq_marlin_repack(qweight.contiguous(), size_k=K, size_n=N, num_bits=4)
        self.sc = mu.marlin_permute_scales(scales.to(dtype).contiguous(), size_k=K, size_n=N, group_size=128)
        self.zp = mu.awq_to_marlin_zero_points(qzeros.contiguous(), size_k=K // 128, size_n=N, num_bits=4)
        self.ws = mu.marlin_make_workspace_new(dev)
        self.g_idx = mu.marlin_make_empty_g_idx(dev)
        self.sort = mu.marlin_make_empty_g_idx(dev)
        self.qt = scalar_types.uint4
        self.apply_fn = mu.apply_awq_marlin_linear

    def __call__(self, x):
        return self.apply_fn(input=x, weight=self.qw, weight_scale=self.sc, weight_zp=self.zp, g_idx=self.g_idx,
                             g_idx_sort_indices=self.sort, workspace=self.ws, quant_type=self.qt,
                             output_size_per_partition=self.N, input_size_per_partition=self.K, bias=None)


class ReferenceLinear:
    """rotate_p -> Marlin_p for every partition, torch.cat (plugin.py:288-311)."""

    def __init__(self, L, dtype, rotate):
        self.rotate = rotate
        self.L = L
        self.parts = []
        n0 = 0
        for n in L.part_sizes:
            self.parts.append(MarlinLinear(L.qweight[:, n0 // 8:(n0 + n) // 8], L.qzeros[:, n0 // 8:(n0 + n) // 8],
                                           L.scales[:, n0:n0 + n], L.in_features, n, dtype))
            n0 += n

    def __call__(self, x):
        outs = []
        for p, ml in enumerate(self.parts):
            xr = self.rotate(x, self.L.pairs[p], self.L.theta[p], self.L.channel_scales[p])
            outs.append(ml(xr))
        return outs[0] if len(outs) == 1 else torch.cat(outs, dim=-1)


def golden(outdir: Path) -> None:
    rotate = load_reference_rotate()
    outdir.mkdir(parents=True, exist_ok=True)
    dev = "cuda"
    # ---- rotate fixtures
    cases = [  # name, dtype, M, K, G, krot, use_scale, uniform_pi
        ("bf16_m1", "bfloat16", 1, 1024, 128, 8, True, False), ("bf16_m5", "bfloat16", 5, 512, 128, 8, True, False),
        ("bf16_m16_pi", "bfloat16", 16, 512, 128, 8, True, True), ("f16_m3", "float16", 3, 512, 128, 8, True, False),
        ("f16_noscale", "float16", 4, 512, 128, 8, False, False), ("f32_m6", "float32", 6, 512, 128, 8, True, False),
        ("bf16_g64_k1", "bfloat16", 7, 256, 64, 1, True, False), ("f32_g64_k8", "float32", 2, 256, 64, 8, False, True),
    ]
    for i, (name, dt, M, K, G, krot, use_scale, pi) in enumerate(cases):
        L = make_synthetic_layer(K, [64], group_size=G, krot=krot, seed=100 + i, theta_uniform_pi=pi)
        x = make_synthetic_activations(M, K, seed=200 + i, dtype=_TD[dt]).to(dev)
        th, pr, cs = L.theta[0].to(dev), L.pairs[0].to(dev), L.channel_scales[0].to(dev)
        out = rotate(x, pr, th, cs if use_scale else None, G)
        rec = dict(dtype=dt, theta_dtype="float16", group=G, x=bits(x), pairs=pr.cpu().numpy(), theta=bits(th), out=bits(out))
        if use_scale:
            rec["scales"] = bits(cs)
        np.savez_compressed(outdir / f"ref_gpu_rotate_{name}.npz", **rec)
    # ---- rotate + Marlin fixtures (merged 2-partition layer), with Marlin's dequantised operand
    for i, (dt, M) in enumerate((("bfloat16", 1), ("bfloat16", 16), ("float16", 4))):
        L = make_synthetic_layer(512, [256, 128], seed=300 + i).to(dev)
        x = make_synthetic_activations(M, 512, seed=400 + i, dtype=_TD[dt]).to(dev)
        ref = ReferenceLinear(L, _TD[dt], rotate)
        y = ref(x)
        rows = torch.tensor([0, 1, 127, 128, 300, 511])
        onehot = torch.zeros(len(rows), 512, dtype=_TD[dt], device=dev)
        onehot[torch.arange(len(rows)), rows] = 1.0
        w_rows = torch.cat([ml(onehot) for ml in ref.parts], dim=-1)     # Marlin only, no rotation
        np.savez_compressed(outdir / f"ref_gpu_linear_{dt}_m{M}.npz", dtype=dt, x=bits(x), qweight=L.qweight.cpu().numpy(),
                            qzeros=L.qzeros.cpu().numpy(), scales=bits(L.scales), theta=bits(L.theta), pairs=L.pairs.cpu().numpy(),
                            channel_scales=bits(L.channel_scales), part_sizes=np.array(L.part_sizes), y=bits(y),
                            w_onehot=bits(w_rows), w_rows=rows.numpy())
    print("golden fixtures written to", outdir)


# seed-defined cases of tests/test_gpu_reference.py: the layer and the activations are regenerated from the seeds there
PIPELINE_CASES = [
    dict(name="rot_bf16", kind="rotate", dtype="bfloat16", M=16, K=4096, parts=[64], seed=1, xseed=2),
    dict(name="rot_f16", kind="rotate", dtype="float16", M=3, K=4096, parts=[64], seed=3, xseed=4),
    dict(name="rot_f32", kind="rotate", dtype="float32", M=5, K=1024, parts=[64], seed=5, xseed=6),
    dict(name="o_m1", kind="linear", dtype="bfloat16", M=1, K=4096, parts=[4096], seed=7, xseed=8),
    dict(name="o_m16", kind="linear", dtype="bfloat16", M=16, K=4096, parts=[4096], seed=7, xseed=9),
    dict(name="qkv_m4", kind="linear", dtype="bfloat16", M=4, K=4096, parts=[4096, 1024, 1024], seed=10, xseed=11),
    dict(name="down_m1_f16", kind="linear", dtype="float16", M=1, K=14336, parts=[4096], seed=12, xseed=13),
    # large M (rotation pre-pass + tensor-core GEMM), incl. K = 11008 / 14336
    dict(name="o_m256", kind="linear", dtype="bfloat16", M=256, K=4096, parts=[4096], seed=7, xseed=14),
    dict(name="o_m1024", kind="linear", dtype="bfloat16", M=1024, K=4096, parts=[4096], seed=7, xseed=15),
    dict(name="qkv_m256", kind="linear", dtype="bfloat16", M=256, K=4096, parts=[4096, 1024, 1024], seed=10, xseed=16),
    dict(name="qkv_m1024", kind="linear", dtype="bfloat16", M=1024, K=4096, parts=[4096, 1024, 1024], seed=10, xseed=17),
    dict(name="l2down_m256", kind="linear", dtype="bfloat16", M=256, K=11008, parts=[4096], seed=18, xseed=19),
    dict(name="l2down_m1024_f16", kind="linear", dtype="float16", M=1024, K=11008, parts=[4096], seed=18, xseed=20),
    dict(name="down_m256", kind="linear", dtype="bfloat16", M=256, K=14336, parts=[4096], seed=12, xseed=21),
    dict(name="down_m1024", kind="linear", dtype="bfloat16", M=1024, K=14336, parts=[4096], seed=12, xseed=22),
    dict(name="gate_up_m16", kind="linear", dtype="bfloat16", M=16, K=4096, parts=[14336, 14336], seed=23, xseed=24),
]
SAMPLE_DRAWS = 4096   # seeded draws of flat indices per case; every 4th of them (sorted) is kept


def samples(out: Path) -> None:
    """Reference outputs of PIPELINE_CASES at a seeded sample of SAMPLE_DRAWS / 4 flat indices, as raw bits: small enough
    to keep under tests/golden/."""
    rotate = load_reference_rotate()
    res = {"spec": json.dumps(PIPELINE_CASES)}
    for i, c in enumerate(PIPELINE_CASES):
        dt = _TD[c["dtype"]]
        L = make_synthetic_layer(c["K"], c["parts"], seed=c["seed"]).to("cuda")
        x = make_synthetic_activations(c["M"], c["K"], seed=c["xseed"], dtype=dt).to("cuda")
        y = rotate(x, L.pairs[0], L.theta[0], L.channel_scales[0]) if c["kind"] == "rotate" else ReferenceLinear(L, dt, rotate)(x)
        flat = bits(y).reshape(-1)
        n = min(flat.size, SAMPLE_DRAWS)
        idx = np.sort(np.random.default_rng(1000 + i).choice(flat.size, n, replace=False))[::4].astype(np.int32)
        res[c["name"] + "_shape"] = np.array(y.shape, dtype=np.int64)
        res[c["name"] + "_idx"] = idx
        res[c["name"] + "_val"] = flat[idx]
    out.parent.mkdir(parents=True, exist_ok=True)
    np.savez_compressed(out, **res)
    print("reference samples written to", out)


def bench(out: Path, ms: list[int]) -> None:
    """Per-linear time of the reference pair (its rotate kernel per partition -> vLLM AWQ-Marlin per partition -> cat,
    plugin.py:288-311) on the Llama-3-8B shapes, like-for-like with tools/microbench.py: distinct weight sets > L2,
    the sweep captured as ONE CUDA graph (no launch overhead), CUDA events around several replays."""
    rotate = load_reference_rotate()
    shapes = {"qkv": (4096, [4096, 1024, 1024]), "o": (4096, [4096]), "gate_up": (4096, [14336, 14336]), "down": (14336, [4096])}
    res = {}
    for name, (K, parts) in shapes.items():
        nsets = max(3, int(400e6 // (K * sum(parts) // 2)) + 1)
        layers = [ReferenceLinear(make_synthetic_layer(K, parts, seed=500 + s, device="cuda"), torch.bfloat16, rotate) for s in range(nsets)]
        for m in ms:
            x = make_synthetic_activations(m, K, seed=7, device="cuda")

            def sweep():
                for l in layers:
                    l(x)

            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                sweep()
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            mode = "cuda_graph"
            try:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    sweep()
                run = g.replay
            except Exception as e:  # report eager numbers rather than nothing
                mode = f"eager ({type(e).__name__})"
                run = sweep
            for _ in range(3):
                run()
            torch.cuda.synchronize()
            iters = 20 if m <= 256 else 5
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                run()
            e1.record()
            torch.cuda.synchronize()
            us = e0.elapsed_time(e1) * 1e3 / (iters * nsets)
            res[f"{name}_m{m}"] = {"shape": name, "M": m, "us_per_linear": us, "weight_sets": nsets, "mode": mode,
                                   "kernels_per_linear": 2 * len(parts) + (1 if len(parts) > 1 else 0),
                                   "tflops": 2.0 * m * K * sum(parts) / us / 1e6}
            print(f"{name:8s} M={m:5d} {us:9.2f} us  ({mode})", flush=True)
        del layers
        torch.cuda.empty_cache()
    out.write_text(json.dumps(res, indent=1))


def rotbench(which: str) -> None:
    """Standalone rotate op, ours vs the reference's kernel (separate processes: same op name): us and GB/s (read + write)."""
    if which == "reference":
        rotate = load_reference_rotate()
    else:
        import paroquant_b200.kernels.cuda  # noqa: F401
        rotate = torch.ops.rotation.rotate
    for K in (4096, 14336):
        L = make_synthetic_layer(K, [64], seed=3, device="cuda")
        for M in (1, 16, 256, 4096):
            x = make_synthetic_activations(M, K, seed=4, device="cuda")
            for _ in range(3):
                rotate(x, L.pairs[0], L.theta[0], L.channel_scales[0])
            torch.cuda.synchronize()
            reps = 200 if M <= 256 else 30
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                rotate(x, L.pairs[0], L.theta[0], L.channel_scales[0])
            e1.record()
            torch.cuda.synchronize()
            us = e0.elapsed_time(e1) * 1e3 / reps
            print(f"rotate[{which:9s}] K={K:5d} M={M:5d} {us:9.2f} us  {2 * M * K * 2 / us / 1e3:8.1f} GB/s", flush=True)


if __name__ == "__main__":
    cmd = sys.argv[1]
    if cmd == "rotbench":
        rotbench(sys.argv[2])
        sys.exit(0)
    if cmd == "golden":
        golden(Path(sys.argv[2]))
    elif cmd == "samples":
        samples(Path(sys.argv[2]))
    elif cmd == "bench":
        bench(Path(sys.argv[2]), [int(v) for v in sys.argv[4].split(",")] if len(sys.argv) > 4 else [1])
