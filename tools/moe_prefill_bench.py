"""Time one MoE expert block at prefill batch sizes: ParoExperts.prefill_step (grouped wgmma GEMMs, six launches, routing on the
device) captured in a CUDA graph, against ParoExperts.__call__ (eager per-expert linears; it synchronises the host, so it cannot
be captured), alternated in the same process on the same seeded routings.

    python tools/moe_prefill_bench.py [--iters 20] [--sets 4] [--T 32,128,512,2048,4096]

Shapes: Qwen3-30B-A3B-shaped (hidden 2048, I 768, 128 experts, top-8) and Mixtral-8x7B-shaped (hidden 4096, I 14336, 8 experts,
top-2).  Synthetic weights generated on the device; `--sets` weight sets are used round-robin so the working set exceeds the
50 MB L2.  TFLOP/s counts the selected experts' work, 2 * sum over valid (token, slot) of (H * 2I + I * H).  The HBM bound counts
the bytes of the experts actually selected (int4 weights, scales, zeros), the two shared rotations, x and y, at the data-sheet
3.35 TB/s.  Times are medians over the iterations, with the 25th / 75th percentiles as the spread.  The GPU's name, power limit
and SM clock are read before and after the timing in the same run.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from paroquant_b200.checkpoint import ParoLayerBuffers, make_synthetic_layer  # noqa: E402
from paroquant_b200.experts import ParoExperts  # noqa: E402

HBM_BPS = 3.35e12
SHAPES = {"qwen3_30b_a3b": (2048, 768, 128, 8), "mixtral_8x7b": (4096, 14336, 8, 2)}


def _experts(E, H, I, seed):
    sg, sd = make_synthetic_layer(H, [I, I], seed=seed, device="cuda"), make_synthetic_layer(I, [H], seed=seed + 1, device="cuda")
    blocks = []
    for e in range(E):
        gu = make_synthetic_layer(H, [I, I], seed=seed + 10 + e, device="cuda")
        d = make_synthetic_layer(I, [H], seed=seed + 500 + e, device="cuda")
        gu = ParoLayerBuffers(gu.qweight, gu.qzeros, gu.scales, sg.theta.clone(), sg.pairs.clone(), sg.channel_scales.clone(), [I, I], 128, None)
        gu.theta[1], gu.pairs[1], gu.channel_scales[1] = gu.theta[0], gu.pairs[0], gu.channel_scales[0]
        blocks.append({"gate_up": gu, "down": ParoLayerBuffers(d.qweight, d.qzeros, d.scales, sd.theta, sd.pairs, sd.channel_scales, [H], 128, None)})
    ex = ParoExperts(blocks, torch.bfloat16)
    del blocks
    return ex


def _work(ids, E, H, I, T):
    valid = (ids >= 0) & (ids < E)
    n_sel = len(torch.unique(ids[valid]))
    per_expert = (H * 2 * I + I * H) // 2 + (H // 128 * 2 * I + I // 128 * H) * 3   # int4 weights + bf16 scales + uint8 zeros
    rot = (H + I) * (8 * 3 + 2)                                                       # pairs, theta, channel scales of both rotations
    nbytes = n_sel * per_expert + rot + T * H * 2 * 2
    flops = 2 * int(valid.sum()) * (H * 2 * I + I * H)
    return flops, nbytes


def _gpu():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:   # report, do not fail the measurement
        return f"unknown ({e})"


def _pct(v, p):
    s = sorted(v)
    return s[min(len(s) - 1, int(p * len(s)))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--sets", type=int, default=4)
    ap.add_argument("--T", default="32,128,512,2048,4096")
    ap.add_argument("--shapes", default=",".join(SHAPES))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("moe_prefill_bench needs a CUDA device")
    print(json.dumps({"gpu_before": _gpu()}), flush=True)
    for name in a.shapes.split(","):
        H, I, E, k = SHAPES[name]
        sets = [_experts(E, H, I, 1000 * s) for s in range(a.sets)]
        for T in (int(t) for t in a.T.split(",")):
            g = torch.Generator(device="cuda").manual_seed(T)
            routes = [torch.rand(T, E, generator=g, device="cuda").topk(k, -1) for _ in range(a.iters)]
            x = torch.randn(T, H, device="cuda", dtype=torch.bfloat16)
            steps = [ex.prefill_step(T, k) for ex in sets]
            graphs = []
            for ex, st in zip(sets, steps):
                st.x.copy_(x)
                st.topk_ids.copy_(routes[0].indices)
                st.topk_weights.copy_(torch.softmax(routes[0].values, -1))
                st.step()
                ex(x, routes[0].indices, torch.softmax(routes[0].values, -1))   # warm the eager path's per-shape state
                s = torch.cuda.Stream()
                s.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(s):
                    st.step()
                torch.cuda.current_stream().wait_stream(s)
                gr = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gr):
                    st.step()
                graphs.append(gr)
            torch.cuda.synchronize()
            new_t, old_t, work = [], [], []
            for it, r in enumerate(routes):
                s = it % a.sets
                w = torch.softmax(r.values, -1)
                steps[s].topk_ids.copy_(r.indices)
                steps[s].topk_weights.copy_(w)
                e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
                e0.record()
                graphs[s].replay()
                e1.record()
                sets[s](x, r.indices, w)
                e2.record()
                torch.cuda.synchronize()
                new_t.append(e0.elapsed_time(e1) * 1e3)
                old_t.append(e1.elapsed_time(e2) * 1e3)
                work.append(_work(r.indices, E, H, I, T))
            med = lambda v: _pct(v, 0.5)   # noqa: E731
            flops, nbytes = med([f for f, _ in work]), med([b for _, b in work])
            tn, to = med(new_t), med(old_t)
            print(json.dumps({
                "shape": name, "T": T, "top_k": k,
                "prefill_step_us": round(tn, 1), "prefill_p25_p75": [round(_pct(new_t, 0.25), 1), round(_pct(new_t, 0.75), 1)],
                "eager_call_us": round(to, 1), "eager_p25_p75": [round(_pct(old_t, 0.25), 1), round(_pct(old_t, 0.75), 1)],
                "speedup": round(to / tn, 2), "prefill_tflops": round(flops / tn / 1e6, 1), "eager_tflops": round(flops / to / 1e6, 1),
                "hbm_bound_us": round(nbytes / HBM_BPS * 1e6, 1), "selected_MB": round(nbytes / 1e6, 1)}), flush=True)
            del steps, graphs
            torch.cuda.empty_cache()
        del sets
        torch.cuda.empty_cache()
    print(json.dumps({"gpu_after": _gpu()}), flush=True)


if __name__ == "__main__":
    main()
