"""Prefill microbenchmark (BASELINE.json config 2): fused rotate + dequant + wgmma GEMM,
batch in {256, 1024, 4096}, Llama shapes; TFLOP/s against the measured bf16 tensor roofline.
    python tools/gemm_bench.py [--out gpurun_out/gemm.json]
"""
import argparse, json, sys
from pathlib import Path
import torch
ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from bench import measured_peaks
from paroquant_b200 import _cabi
from paroquant_b200.checkpoint import make_synthetic_activations, make_synthetic_layer
from paroquant_b200.linear import ParoLinearKernel

SHAPES = {"q_o": (4096, [4096]), "qkv": (4096, [4096, 1024, 1024]), "gate_up": (4096, [14336, 14336]), "down": (14336, [4096]),
          "l2_up": (4096, [11008]), "l2_down": (11008, [4096])}

def run(name, M, reps=10):
    K, parts = SHAPES[name]
    k = ParoLinearKernel.from_buffers(make_synthetic_layer(K, parts, seed=3, device="cuda"), torch.bfloat16, check_pairs=False, max_m=M)
    x = make_synthetic_activations(M, K, seed=1, device="cuda")
    y = torch.empty(M, sum(parts), dtype=torch.bfloat16, device="cuda")
    for _ in range(3):
        _cabi.linear_forward(k.shape, k.packed, x, None, k.workspace, out=y)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        _cabi.linear_forward(k.shape, k.packed, x, None, k.workspace, out=y)
    e1.record(); torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / reps
    fl = 2.0 * M * K * sum(parts)
    _, tf_peak, src = measured_peaks()
    return {"shape": name, "M": M, "us": us, "TFLOPs": fl / us / 1e6, "frac_tensor": fl / us / 1e6 / tf_peak, "peak_source": src, "launches": _cabi.last_launch_count()}

if __name__ == "__main__":
    ap = argparse.ArgumentParser(); ap.add_argument("--out", default=""); ap.add_argument("--ms", default="256,1024,4096"); ap.add_argument("--shapes", default="q_o,gate_up,down")
    a = ap.parse_args(); res = []
    for n in a.shapes.split(","):
        for M in [int(v) for v in a.ms.split(",")]:
            r = run(n, M); res.append(r)
            print(f"{n:10s} M={M:5d} {r['us']:9.1f} us {r['TFLOPs']:8.1f} TFLOP/s {100*r['frac_tensor']:5.1f}% of {r['peak_source']} bf16 peak ({r['launches']} launches)", flush=True)
            torch.cuda.empty_cache()
    if a.out: Path(a.out).write_text(json.dumps(res, indent=1))
