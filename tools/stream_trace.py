"""In-kernel timeline of the small-M kernel (PARO_DECODE_TRACE=1): SM cycles since kernel entry, per step.

    PARO_DECODE_TRACE=1 python tools/stream_trace.py [--shape gate_up] [--m 1] [--chain]

slots: 0 before griddepcontrol.wait | 1 step start | 2 dependency flag passed | 3 B operand ready | 4 first record
landed | 5 my rounds done (worker warp 0) | 6 epilogue group done | 7 last D read back | 8 last block counter
answered | 9 last fix-up: slots being added.  Printed: CTA 0, median, max over the CTAs.
"""
from __future__ import annotations

import argparse
import ctypes
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from paroquant_b200 import _cabi, chain  # noqa: E402
from paroquant_b200.checkpoint import make_synthetic_activations, make_synthetic_layer  # noqa: E402
from paroquant_b200.linear import ParoLinearKernel  # noqa: E402

H, KV, I = 4096, 1024, 14336
SH = {"o": (H, [H]), "gate_up": (H, [I, I]), "down": (I, [H]), "qkv": (H, [H, KV, KV])}
NAMES = ["before pdl wait", "step start", "flag passed", "B operand ready", "first record", "rounds done", "epilogue done",
         "last D read", "last D full", "last fix-up", "-", "pass 1 start"]


def dump(nsteps):
    nct, nst, nsl = torch.cuda.get_device_properties(0).multi_processor_count, 6, 12
    buf = (ctypes.c_ulonglong * (nct * nst * nsl))()
    assert _cabi.lib().paro_debug_stream_trace(buf, nct) == 0
    t = torch.tensor(list(buf), dtype=torch.float64).view(nct, nst, nsl)
    for i in range(nsteps):
        print(f" step {i}:   {'CTA 0':>8s} {'median':>8s} {'max':>8s}")
        for sl in range(12):
            col = t[:, i, sl]
            print(f"   {NAMES[sl]:16s} {int(col[0]):8d} {int(col.median()):8d} {int(col.max()):8d}")
        order = torch.argsort(t[:, i, 6], descending=True)
        pick = [int(v) for v in order[:4]] + [int(order[len(order) // 2])]
        print("   rows (slowest 4 CTAs by epilogue done, then the median one): cta | " + " | ".join(n.split()[-1] for n in NAMES))
        for c in pick:
            print(f"   cta {c:3d}: " + " ".join(f"{int(v):7d}" for v in t[c, i]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", default="gate_up")
    ap.add_argument("--m", type=int, default=1)
    ap.add_argument("--chain", action="store_true")
    a = ap.parse_args()
    M, dt, dev = a.m, torch.bfloat16, "cuda"
    if a.chain:
        ks = [{n: ParoLinearKernel.from_buffers(make_synthetic_layer(K, p, seed=500 + 8 * li + i, device=dev), dt, check_pairs=False, max_m=M)
               for i, (n, (K, p)) in enumerate(SH.items())} for li in range(3)]
        attn = make_synthetic_activations(M, H, seed=1, device=dev, dtype=dt)
        resid = make_synthetic_activations(M, H, seed=2, device=dev, dtype=dt)
        w = torch.ones(H, dtype=dt, device=dev)
        chains = [chain.decoder_tail(l["o"], l["gate_up"], l["down"], l["qkv"], attn_out=attn, residual=resid, post_attn_norm=w, next_input_norm=w)[0]
                  for l in ks]
        for _ in range(3):
            for c in chains:
                c()
        torch.cuda.synchronize()
        print(f"chain o -> gate_up -> down -> qkv, M={M} (third of three back-to-back launches on cold weights)")
        dump(4)
        return
    K, parts = SH[a.shape]
    ks = [ParoLinearKernel.from_buffers(make_synthetic_layer(K, parts, seed=900 + i, device=dev), dt, check_pairs=False, max_m=M) for i in range(4)]
    x = make_synthetic_activations(M, K, seed=1, device=dev, dtype=dt)
    for _ in range(3):
        for k in ks:
            k(x)
    torch.cuda.synchronize()
    print(f"{a.shape} M={M} (last of back-to-back launches)")
    dump(1)


if __name__ == "__main__":
    main()
