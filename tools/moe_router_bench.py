"""Time a MoE block from hidden state to block output with the routing computed on the device by the library
(ParoExperts.decode_step / prefill_step with router=ParoRouter: 3 / 7 launches) against the same block fed by torch routing
(F.linear -> softmax -> topk -> renormalise -> two copy_ into the step's buffers, then the block's 2 / 6 launches).  Both are
captured as one CUDA graph each and replayed alternately in the same process on the same inputs; medians are reported.

    python tools/moe_router_bench.py [--iters 50] [--sets 4] [--T 1,4,16,32,512,4096] [--shapes qwen3_30b_a3b,mixtral_8x7b]

Shapes: Qwen3-30B-A3B-shaped (hidden 2048, I 768, 128 experts, top-8) and Mixtral-8x7B-shaped (hidden 4096, I 14336, 8 experts,
top-2); T <= 16 runs decode_step, larger T prefill_step.  Synthetic weights generated on the device; `--sets` weight sets (experts
and router) are used round-robin so the working set exceeds the 50 MB L2.  The router launch alone is timed as a graph of one
launch per weight set, divided by the sets.  Its bound counts the bytes of the router weight and x once, at the data-sheet
3.35 TB/s: at these sizes (64 KB to 512 KB of weight) that bound is a fraction of a microsecond and the launch is latency, not
bandwidth -- the share says how far from the bound, not how well HBM is used.  The GPU's name, power limit and SM clock are read
before and after the timing in the same run.  Needs a CUDA device.
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
from paroquant_b200.experts import ParoExperts, ParoRouter  # noqa: E402

HBM_BPS = 3.35e12
SHAPES = {"qwen3_30b_a3b": (2048, 768, 128, 8), "mixtral_8x7b": (4096, 14336, 8, 2)}
DT = torch.bfloat16


def _experts(E, H, I, seed):
    sg, sd = make_synthetic_layer(H, [I, I], seed=seed, device="cuda"), make_synthetic_layer(I, [H], seed=seed + 1, device="cuda")
    blocks = []
    for e in range(E):
        gu = make_synthetic_layer(H, [I, I], seed=seed + 10 + e, device="cuda")
        d = make_synthetic_layer(I, [H], seed=seed + 500 + e, device="cuda")
        gu = ParoLayerBuffers(gu.qweight, gu.qzeros, gu.scales, sg.theta.clone(), sg.pairs.clone(), sg.channel_scales.clone(), [I, I], 128, None)
        gu.theta[1], gu.pairs[1], gu.channel_scales[1] = gu.theta[0], gu.pairs[0], gu.channel_scales[0]
        blocks.append({"gate_up": gu, "down": ParoLayerBuffers(d.qweight, d.qzeros, d.scales, sd.theta, sd.pairs, sd.channel_scales, [H], 128, None)})
    ex = ParoExperts(blocks, DT)
    del blocks
    return ex


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


def _capture(fn):
    """fn warmed on a side stream, then captured."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fn()
    return graph


def _torch_routed(step, w, k):
    def run():
        p = torch.softmax(torch.nn.functional.linear(step.x, w).float(), -1)
        tw, ti = torch.topk(p, k, dim=-1)
        step.topk_ids.copy_(ti)
        step.topk_weights.copy_(tw / tw.sum(-1, keepdim=True))
        step.step()
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--sets", type=int, default=4)
    ap.add_argument("--T", default="1,4,16,32,512,4096")
    ap.add_argument("--shapes", default=",".join(SHAPES))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("moe_router_bench needs a CUDA device")
    print(json.dumps({"gpu_before": _gpu()}), flush=True)
    for name in a.shapes.split(","):
        H, I, E, k = SHAPES[name]
        sets = [_experts(E, H, I, 1000 * s) for s in range(a.sets)]
        g = torch.Generator(device="cuda").manual_seed(E)
        routers = [ParoRouter(torch.randn(E, H, generator=g, device="cuda") * (2.0 / H ** 0.5), k, True, dtype=DT) for _ in sets]
        for T in (int(t) for t in a.T.split(",")):
            xs = [torch.randn(T, H, generator=g, device="cuda").to(DT) for _ in range(a.iters)]
            make = (lambda ex, **kw: ex.decode_step(T, k, **kw)) if T <= 16 else (lambda ex, **kw: ex.prefill_step(T, k, **kw))
            dev_steps = [make(ex, router=r) for ex, r in zip(sets, routers)]
            torch_steps = [make(ex) for ex in sets]
            for st in dev_steps + torch_steps:
                st.x.copy_(xs[0])
            dev_graphs = [_capture(st.step) for st in dev_steps]
            torch_graphs = [_capture(_torch_routed(st, r.weight, k)) for st, r in zip(torch_steps, routers)]

            def all_routers():
                for st in dev_steps:
                    st._route()
            router_graph = _capture(all_routers)
            torch.cuda.synchronize()
            dev_t, torch_t, router_t, same = [], [], [], 0
            for it, x in enumerate(xs):
                s = it % a.sets
                dev_steps[s].x.copy_(x)
                torch_steps[s].x.copy_(x)
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
                order = (dev_graphs[s], torch_graphs[s]) if it % 2 == 0 else (torch_graphs[s], dev_graphs[s])
                ev[0].record()
                order[0].replay()
                ev[1].record()
                order[1].replay()
                ev[2].record()
                router_graph.replay()
                ev[3].record()
                torch.cuda.synchronize()
                first, second = ev[0].elapsed_time(ev[1]) * 1e3, ev[1].elapsed_time(ev[2]) * 1e3
                dev_t.append(first if it % 2 == 0 else second)
                torch_t.append(second if it % 2 == 0 else first)
                router_t.append(ev[2].elapsed_time(ev[3]) * 1e3 / a.sets)
                same += int(torch.equal(dev_steps[s].topk_ids.sort(-1).values, torch_steps[s].topk_ids.int().sort(-1).values))
            med = lambda v: _pct(v, 0.5)   # noqa: E731
            bound = (E * H * 2 + T * H * 2) / HBM_BPS * 1e6
            print(json.dumps({
                "shape": name, "T": T, "top_k": k, "path": "decode_step" if T <= 16 else "prefill_step",
                "device_routed_us": round(med(dev_t), 2), "device_p25_p75": [round(_pct(dev_t, 0.25), 2), round(_pct(dev_t, 0.75), 2)],
                "torch_routed_us": round(med(torch_t), 2), "torch_p25_p75": [round(_pct(torch_t, 0.25), 2), round(_pct(torch_t, 0.75), 2)],
                "torch_over_device": round(med(torch_t) / med(dev_t), 3),
                "router_alone_us": round(med(router_t), 2), "router_hbm_bound_us": round(bound, 3),
                "router_share_of_bound": round(bound / med(router_t), 3),
                "steps_with_same_expert_sets": f"{same}/{len(xs)}"}), flush=True)
            del dev_steps, torch_steps, dev_graphs, torch_graphs, router_graph
            torch.cuda.empty_cache()
        del sets, routers
        torch.cuda.empty_cache()
    print(json.dumps({"gpu_after": _gpu()}), flush=True)


if __name__ == "__main__":
    main()
