"""Decoder-tail chain vs the same four linears launched one by one (Llama-3-8B shapes, decode batch M).

    python tools/chain_bench.py [--m 1] [--layers 6] [--trace]

Per layer: o 4096->4096, gate_up 4096->28672, down 14336->4096, (next) qkv 4096->6144 = 114.5 MB of packed weights;
`--layers` distinct weight sets are cycled (>= 4 keeps the working set above the 126 MB L2).  Both variants run as a
CUDA graph (PDL edges on).  The per-linear variant launches only the linears (no norm / activation kernels), i.e. it is
the lower bound of the unfused path.  With --trace the in-kernel timeline of CTA 0 / the slowest CTA is printed.
"""
from __future__ import annotations

import argparse
import ctypes
import os
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from bench import algorithmic_bytes, measured_peaks  # noqa: E402
from paroquant_b200 import _cabi, chain  # noqa: E402
from paroquant_b200.checkpoint import make_synthetic_activations, make_synthetic_layer  # noqa: E402
from paroquant_b200.linear import ParoLinearKernel  # noqa: E402

H, KV, I = 4096, 1024, 14336
SH = {"o": (H, [H]), "gate_up": (H, [I, I]), "down": (I, [H]), "qkv": (H, [H, KV, KV])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--m", type=int, default=1)
    ap.add_argument("--layers", type=int, default=6)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--trace", action="store_true")
    a = ap.parse_args()
    M, dt, dev = a.m, torch.bfloat16, "cuda"
    layers = []
    for li in range(a.layers):
        layers.append({n: ParoLinearKernel.from_buffers(make_synthetic_layer(K, p, seed=500 + 8 * li + i, device=dev), dt, check_pairs=False, max_m=M)
                       for i, (n, (K, p)) in enumerate(SH.items())})
    attn = make_synthetic_activations(M, H, seed=1, device=dev, dtype=dt)
    resid = make_synthetic_activations(M, H, seed=2, device=dev, dtype=dt)
    w = torch.ones(H, dtype=dt, device=dev)
    chains = [chain.decoder_tail(l["o"], l["gate_up"], l["down"], l["qkv"], attn_out=attn, residual=resid, post_attn_norm=w, next_input_norm=w)
              for l in layers]
    xs = {n: make_synthetic_activations(M, K, seed=3 + i, device=dev, dtype=dt) for i, (n, (K, p)) in enumerate(SH.items())}
    ys = {n: torch.empty(M, sum(p), dtype=dt, device=dev) for n, (K, p) in SH.items()}

    def run_chain():
        for c, _ in chains:
            c()

    def run_single():
        for l in layers:
            for n in SH:
                k = l[n]
                _cabi.linear_forward(k.shape, k.packed, xs[n], None, k.workspace, out=ys[n])

    layer_bytes = sum(algorithmic_bytes(K, p, M) for K, p in SH.values())
    peak, _, src = measured_peaks()
    for name, fn in (("chain", run_chain), ("single", run_single)):
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            fn()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fn()
        for _ in range(3):
            g.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.reps):
            g.replay()
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / (a.reps * a.layers)
        print(f"{name:7s} M={M:2d}  {us:7.2f} us / layer   {layer_bytes / us / 1e3:6.0f} GB/s  {100 * layer_bytes / us / 1e3 / peak:5.1f}% of {src} HBM"
              f"   -> {1e6 / (32 * us) * M:7.0f} tok/s for 32 layers", flush=True)
    if a.trace:
        if os.environ.get("PARO_DECODE_TRACE") != "1":
            print("set PARO_DECODE_TRACE=1 for the timeline")
            return
        chains[0][0]()
        torch.cuda.synchronize()
        nct, nst, nsl = torch.cuda.get_device_properties(0).multi_processor_count, 6, 8
        buf = (ctypes.c_ulonglong * (nct * nst * nsl))()
        assert _cabi.lib().paro_debug_stream_trace(buf, nct) == 0
        t = torch.tensor(list(buf), dtype=torch.float64).view(nct, nst, nsl)
        names = ["entry->pdl", "step start", "flag passed", "xb ready", "first record", "rounds done", "epilogue done", "-"]
        print("cycles since kernel entry (CTA 0 | median | max over CTAs), per step")
        for i in range(4):
            print(f" step {i}")
            for sl in range(7):
                col = t[:, i, sl]
                print(f"   {names[sl]:14s} {int(col[0]):8d} {int(col.median()):8d} {int(col.max()):8d}")


if __name__ == "__main__":
    main()
