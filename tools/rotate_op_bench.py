"""torch.ops.rotation.rotate forward times, CUDA events, one JSON line:
- the forward column of tools/backward_bench.py (five training shapes, krot 8);
- bf16 at M = 1 and 16, K = 4096: one CUDA graph of `--calls` rotate launches, so a call's time is its device time between
  dependent launches (where fetching the rotations' pair words and angles, not HBM, sets the time).

    python tools/rotate_op_bench.py [--calls 200] [--reps 20]
"""
import argparse
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import paroquant_b200.kernels.cuda  # noqa: F401,E402
from paroquant_b200.checkpoint import make_synthetic_layer  # noqa: E402
from tools.backward_bench import SHAPES, timed  # noqa: E402


def graph_us(fn, calls, reps):
    """Time per call of `calls` back-to-back launches of fn, captured as one CUDA graph and replayed `reps` times."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(calls):
            fn()
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (reps * calls)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    res = {"gpu": torch.cuda.get_device_name(dev), "training": [], "graph_bf16_k4096": []}
    for dt, M, K, G in SHAPES:
        L = make_synthetic_layer(K, [64], group_size=G, seed=5, device=dev)
        pr, th, sc = L.pairs[0], L.theta[0].float(), L.channel_scales[0].float().view(-1)
        x = torch.randn(M, K, device=dev).to(dt)
        us = timed(lambda: torch.ops.rotation.rotate(x, pr, th, sc, G), reps=a.reps)
        res["training"].append({"dtype": str(dt).replace("torch.", ""), "M": M, "K": K, "G": G, "forward_us": round(us, 2)})
    L = make_synthetic_layer(4096, [64], seed=5, device=dev)
    pr, th, sc = L.pairs[0], L.theta[0].to(torch.bfloat16), L.channel_scales[0].to(torch.bfloat16).view(-1)
    for M in (1, 16):
        x = torch.randn(M, 4096, device=dev).to(torch.bfloat16)
        us = graph_us(lambda: torch.ops.rotation.rotate(x, pr, th, sc, 128), a.calls, a.reps)
        res["graph_bf16_k4096"].append({"M": M, "us_per_call": round(us, 3)})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
