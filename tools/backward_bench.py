"""Training-side op (SURVEY 8(f) rank 4): forward rotate, the fused backward launch (paro_rotate_backward) and the reference's
backward STRUCTURE -- a Python walk over the rotations, per rotation two one-rotation rotate launches, gathers and a row
reduction (/root/reference/paroquant/kernels/cuda/autograd.py:20-61) -- run on OUR rotate kernel, same box, CUDA events.

    python tools/backward_bench.py [--out backward_bench.json]
"""
import argparse
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import paroquant_b200.kernels.cuda  # noqa: F401,E402
from paroquant_b200 import _cabi  # noqa: E402
from paroquant_b200.checkpoint import make_synthetic_layer  # noqa: E402


# (dtype, M, K, group): the training shapes, also the forward column of tools/rotate_op_bench.py
SHAPES = ((torch.float32, 4096, 4096, 128), (torch.bfloat16, 4096, 4096, 128), (torch.float32, 14336, 4096, 128),
          (torch.float32, 4096, 4096, 64), (torch.float32, 256, 4096, 128))


def stagewise(x, idx_ij, theta, y, grad_out, scale, G):
    krot, K = idx_ij.shape
    rows = y.numel() // K
    t, g = y.reshape(rows, K), grad_out.reshape(rows, K).contiguous()
    base = (torch.arange(K, device=idx_ij.device) // G * G).view(K // 2, 2)[:, 0]
    grad_theta = torch.zeros(krot, K // 2, dtype=torch.float32, device=y.device)
    for r in reversed(range(krot)):
        pr = idx_ij[r].view(K // 2, 2).long()
        ci, cj = pr[:, 0] + base, pr[:, 1] + base
        grad_theta[r] = (g[:, ci].float() * t[:, cj].float() - g[:, cj].float() * t[:, ci].float()).sum(0)
        inv = -theta[r:r + 1]
        t = torch.ops.rotation.rotate(t, idx_ij[r:r + 1], inv, None, G)
        g = torch.ops.rotation.rotate(g, idx_ij[r:r + 1], inv, None, G)
    return (g.float() * scale.float()).to(x.dtype), grad_theta, (x.reshape(rows, K).float() * g.float()).sum(0)


def timed(fn, reps=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / reps


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    res = []
    for dt, M, K, G in SHAPES:
        L = make_synthetic_layer(K, [64], group_size=G, seed=5, device="cuda")
        pr, th, sc = L.pairs[0], L.theta[0].float(), L.channel_scales[0].float().view(-1)
        x = torch.randn(M, K, device="cuda").to(dt)
        go = torch.randn(M, K, device="cuda").to(dt)
        y = torch.ops.rotation.rotate(x, pr, th, sc, G)
        fwd = timed(lambda: torch.ops.rotation.rotate(x, pr, th, sc, G))
        fused = timed(lambda: _cabi.rotate_backward(y, go, x, pr, th, sc, G))
        walk = timed(lambda: stagewise(x, pr, th, y, go, sc, G), reps=5)
        nbytes = M * K * x.element_size()
        r = {"dtype": str(dt).replace("torch.", ""), "M": M, "K": K, "group": G, "forward_us": fwd, "fused_backward_us": fused,
             "stagewise_walk_us": walk, "speedup": walk / fused, "fused_backward_GBps": 4 * nbytes / fused / 1e3}   # reads y, dL/dy, x; writes dL/dx
        res.append(r)
        print(f"{r['dtype']:9s} M={M:6d} K={K} G={G:3d}: forward {fwd:8.1f} us, fused backward {fused:8.1f} us ({r['fused_backward_GBps']:.0f} GB/s), "
              f"stage-wise walk {walk:9.1f} us  -> {r['speedup']:.1f}x", flush=True)
    if a.out:
        Path(a.out).write_text(json.dumps(res, indent=1))
