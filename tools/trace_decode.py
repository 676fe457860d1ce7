"""Phase timeline of the fused small-M kernel (developer aid; needs PARO_DECODE_TRACE=1).
    PARO_DECODE_TRACE=1 python tools/trace_decode.py q_o 1
"""
import ctypes, os, sys
from pathlib import Path
import numpy as np
import torch
ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
os.environ["PARO_DECODE_TRACE"] = "1"
from paroquant_b200 import _cabi
from paroquant_b200.checkpoint import make_synthetic_activations, make_synthetic_layer
from paroquant_b200.linear import ParoLinearKernel
from tools.microbench import SHAPES

name = sys.argv[1] if len(sys.argv) > 1 else "q_o"
M = int(sys.argv[2]) if len(sys.argv) > 2 else 1
K, parts = SHAPES[name]
ks = [ParoLinearKernel.from_buffers(make_synthetic_layer(K, parts, seed=900 + i, device="cuda"), torch.bfloat16, check_pairs=False, max_m=M) for i in range(6)]
x = make_synthetic_activations(M, K, seed=1, device="cuda")
y = torch.empty(M, sum(parts), dtype=torch.bfloat16, device="cuda")
for k in ks:
    _cabi.linear_forward(k.shape, k.packed, x, None, k.workspace, out=y)
torch.cuda.synchronize()
buf = np.zeros(1024 * 12, dtype=np.uint64)
_cabi.lib().paro_debug_trace(buf.ctypes.data_as(ctypes.c_void_p), 1024)
t = buf.reshape(1024, 12)
rounds = buf[200 * 12:200 * 12 + 300].reshape(100, 3).astype(np.int64)
t = t[:200]
t = t[t[:, 10] > 0]
print(f"{name} M={M}: {len(t)} CTAs traced (last launch of a back-to-back chain of 6)")
names = ["", "init+sync", "meta+sincos", "pdl_wait", "rotate+frags", "first stage landed", "main loop", "cluster barrier / atomics", "final reduce+store"]
prev = np.zeros(len(t))
for i in range(1, 9):
    cur = t[:, i].astype(np.float64)
    ok = cur > 0
    d = (cur - prev)[ok]
    if len(d):
        print(f"  {names[i]:28s} +{np.median(d):9.0f} cyc median  (min {d.min():8.0f}  max {d.max():8.0f})   cumulative median {np.median(cur[ok]):9.0f}")
    prev = np.where(ok, cur, prev)
if t[:, 9].max() > 0:
    print(f"  (one-CTA-per-SM kernel) warp 0's last rotation task: x loaded+scaled at {np.median(t[:, 0]):.0f}, rotated rows written at {np.median(t[:, 9]):.0f} (cumulative cycles, median)")
g0, g1 = t[:, 10].astype(np.int64), t[:, 11].astype(np.int64)
print(f"  globaltimer: first entry -> last exit {(g1.max() - g0.min())} ns; entry spread {g0.max() - g0.min()} ns; per-CTA duration median {np.median(g1 - g0):.0f} ns")

if rounds[:, 0].max() > 0:
    print("  CTA 0 per-round log (cycles since entry): round: copy issued / seen full by its set / consumed   [full - issued]")
    for r in range(100):
        if rounds[r, 1] == 0 and rounds[r, 0] == 0:
            break
        print(f"    {r:3d}: {rounds[r,0]:7d} {rounds[r,1]:7d} {rounds[r,2]:7d}   [{rounds[r,1]-rounds[r,0]:6d}]")
