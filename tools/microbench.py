"""Per-shape microbenchmark of the fused small-M kernel (BASELINE.json config 1):
Llama-3-8B q/k/v/o/mlp shapes, batch in {1,4,16}, HBM GB/s against the measured roofline.

    python tools/microbench.py [--out micro.json] [--ms 1,4,16] [--shapes q_o,qkv,...] [--sets N]

Each shape is timed over enough distinct weight sets to exceed the 50 MB L2 (>= 400 MB), as a
CUDA graph of back-to-back launches (PDL on), CUDA events around several replays.  --sets 1 cycles one
weight set that stays in L2 instead (graph of the same length): the kernel's own cost per record without
the HBM stream.  Streaming time close to the L2-resident time means the consumer round, not HBM, is the limit.
Environment knobs forwarded to the library: PARO_DECODE_STAGES, PARO_DECODE_CTAS_PER_SM, PARO_NO_PDL.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from bench import algorithmic_bytes, measured_peaks  # noqa: E402
from paroquant_b200 import _cabi  # noqa: E402
from paroquant_b200.checkpoint import make_synthetic_activations, make_synthetic_layer  # noqa: E402
from paroquant_b200.linear import ParoLinearKernel  # noqa: E402

SHAPES = {"q_o": (4096, [4096]), "kv": (4096, [1024]), "qkv": (4096, [4096, 1024, 1024]), "gate_up": (4096, [14336, 14336]),
          "gate": (4096, [14336]), "down": (14336, [4096]), "qwen_gate_up": (4096, [12288, 12288]), "qwen_down": (12288, [4096]),
          "l2_up": (4096, [11008]), "l2_down": (11008, [4096])}


def time_shape(name, M, reps=20, graph=True, group=128, sets=0):
    K, parts = SHAPES[name]
    wbytes = K * sum(parts) // 2
    launches = max(3, int(400e6 // wbytes) + 1)   # per graph replay
    nsets = sets if sets > 0 else launches
    ks = [ParoLinearKernel.from_buffers(make_synthetic_layer(K, parts, group_size=group, seed=900 + i, device="cuda"), torch.bfloat16,
                                        check_pairs=False, max_m=M) for i in range(nsets)]
    x = make_synthetic_activations(M, K, seed=1, device="cuda")
    y = torch.empty(M, sum(parts), dtype=torch.bfloat16, device="cuda")

    def sweep():
        for i in range(launches):
            k = ks[i % nsets]
            _cabi.linear_forward(k.shape, k.packed, x, None, k.workspace, out=y)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        sweep()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    if graph:
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            sweep()
        run = g.replay
    else:
        run = sweep
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        run()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / (reps * launches)
    ab = algorithmic_bytes(K, parts, M)
    peak, _, src = measured_peaks()
    return {"shape": name, "K": K, "parts": parts, "M": M, "us": us, "alg_bytes": ab, "GBps": ab / us / 1e3,
            "frac_hbm": ab / us / 1e3 / peak, "weight_sets": nsets, "launches": launches, "peak_source": src}


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--ms", default="1,4,16")
    ap.add_argument("--shapes", default="q_o,kv,qkv,gate_up,down")
    ap.add_argument("--no-graph", action="store_true")
    ap.add_argument("--group", type=int, default=128, help="quantisation / rotation group size (64: two scale / zero sets per record)")
    ap.add_argument("--sets", type=int, default=0,
                    help="weight sets cycled through (default: enough to exceed L2, i.e. streamed from HBM); 1: one set that stays in L2, "
                         "which separates the kernels' own per-record cost from HBM bandwidth")
    a = ap.parse_args()
    res = []
    for name in a.shapes.split(","):
        for M in [int(v) for v in a.ms.split(",")]:
            r = time_shape(name, M, graph=not a.no_graph, group=a.group, sets=a.sets)
            res.append(r)
            print(f"{name:12s} M={M:3d} sets={r['weight_sets']:3d} {r['us']:8.2f} us  {r['GBps']:7.0f} GB/s  {100 * r['frac_hbm']:5.1f}% of {r['peak_source']} HBM", flush=True)
            torch.cuda.empty_cache()
    if a.out:
        Path(a.out).write_text(json.dumps(res, indent=1))
