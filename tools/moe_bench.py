"""Time one MoE expert block per decode step: ParoExperts.decode_step (two launches, routing on the device) captured in a CUDA
graph, against ParoExperts.__call__ (eager per-expert chains; it synchronises the host, so it cannot be captured), alternated
in the same process on the same routings.

    python tools/moe_bench.py [--iters 50] [--sets 4]

Shapes: Qwen3-30B-A3B-shaped (hidden 2048, I 768, 128 experts, top-8) and Mixtral-8x7B-shaped (hidden 4096, I 14336, 8 experts,
top-2), T in {1, 4, 16}.  Synthetic weights; `--sets` layers' weight sets are used round-robin so the working set exceeds the
50 MB L2.  Routings are seeded and generated on the device up front.  The HBM bound counts the bytes of the experts actually
selected (weights, scales, zeros), the two shared rotation sets once, and x, ids, weights and y, at the data-sheet 3.35 TB/s.
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


def _experts(E, H, I, seed):
    sg, sd = make_synthetic_layer(H, [I, I], seed=seed), make_synthetic_layer(I, [H], seed=seed + 1)
    blocks = []
    for e in range(E):
        gu, d = make_synthetic_layer(H, [I, I], seed=seed + 10 + e), make_synthetic_layer(I, [H], seed=seed + 500 + e)
        gu = ParoLayerBuffers(gu.qweight, gu.qzeros, gu.scales, sg.theta.clone(), sg.pairs.clone(), sg.channel_scales.clone(), [I, I], 128, None)
        gu.theta[1], gu.pairs[1], gu.channel_scales[1] = gu.theta[0], gu.pairs[0], gu.channel_scales[0]
        blocks.append({"gate_up": gu, "down": ParoLayerBuffers(d.qweight, d.qzeros, d.scales, sd.theta, sd.pairs, sd.channel_scales, [H], 128, None)})
    return ParoExperts(blocks, torch.bfloat16)


def _bytes(ids, E, H, I, T, k):
    n = len(torch.unique(ids[(ids >= 0) & (ids < E)]))
    per_expert = (H * 2 * I + I * H) // 2 + (H // 128 * 2 * I + I // 128 * H) * 3    # int4 weights + bf16 scales + uint8 zeros
    rot = (H + I) * (8 * 3 + 2)                                                        # pairs, theta, channel scales of both rotations
    return n * per_expert + rot + T * H * 2 * 2 + T * k * 8


def _clock():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:   # report, do not fail the measurement
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--sets", type=int, default=4)
    a = ap.parse_args()
    print(json.dumps({"gpu": _clock()}))
    for name, (H, I, E, k) in {"qwen3_30b_a3b": (2048, 768, 128, 8), "mixtral_8x7b": (4096, 14336, 8, 2)}.items():
        sets = [_experts(E, H, I, 1000 * s) for s in range(a.sets)]
        for T in (1, 4, 16):
            g = torch.Generator(device="cuda").manual_seed(T)
            routes = [torch.rand(T, E, generator=g, device="cuda").topk(k, -1) for _ in range(a.iters)]
            steps = [ex.decode_step(T, k) for ex in sets]
            x = torch.randn(T, H, device="cuda", dtype=torch.bfloat16)
            graphs = []
            for st in steps:
                st.x.copy_(x)
                st.topk_ids.copy_(routes[0].indices)
                st.topk_weights.copy_(torch.softmax(routes[0].values, -1))
                st.step()
                gr = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gr):
                    st.step()
                graphs.append(gr)
            torch.cuda.synchronize()
            new_t, old_t, nbytes = [], [], []
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
                nbytes.append(_bytes(r.indices, E, H, I, T, k))
            med = lambda v: sorted(v)[len(v) // 2]   # noqa: E731
            bound = med(nbytes) / HBM_BPS * 1e6
            print(json.dumps({"shape": name, "T": T, "decode_step_us": round(med(new_t), 2), "eager_call_us": round(med(old_t), 2),
                              "hbm_bound_us": round(bound, 2), "share_of_bound": round(bound / med(new_t), 3),
                              "selected_MB": round(med(nbytes) / 1e6, 1)}))
        del sets, steps, graphs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
