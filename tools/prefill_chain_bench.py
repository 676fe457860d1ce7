"""Time a Llama-3-8B decoder tail above 16 rows: the prefill chain (ParoPrefillChain, decoder_tail for m > 16: per linear a
rotation pre-pass with the x op folded in and an INT4 wgmma GEMM with the residual epilogue) against the unfused path (one
ParoLinearKernel.forward_into per linear, torch residual add / RMSNorm / SiLU * up between them, written as in
tests/test_gpu_chain.py).  Both are captured in CUDA graphs and alternated in the same process.

    python tools/prefill_chain_bench.py [--iters 20] [--sets 2] [--M 32,64,128,256,1024,4096]

The tail is o (4096 -> 4096) + residual, RMSNorm -> gate_up (4096 -> 2 x 14336) -> SiLU * up -> down (14336 -> 4096) + residual,
RMSNorm -> next qkv (4096 -> 4096 + 1024 + 1024), bf16 activations, group 128, krot 8.  Synthetic weights are generated on the
device; `--sets` weight sets (about 110 MB of packed weights each) are used round-robin so the working set exceeds the 50 MB L2.
TFLOP/s counts 2 * M * (sum of K * N of the four linears).  Launches per block are counted by torch.profiler on one eager call
of each variant.  The two variants' outputs are compared (normwise relative error of every buffer, limit 1e-3).  Times are
medians over the iterations, with the 25th / 75th percentiles as the spread.  The GPU's name, power limit and SM clock are read
before and after the timing in the same run.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from paroquant_b200 import _cabi, chain  # noqa: E402
from paroquant_b200.checkpoint import make_synthetic_layer  # noqa: E402
from paroquant_b200.linear import ParoLinearKernel  # noqa: E402

H, I, QKV = 4096, 14336, [4096, 1024, 1024]
EPS = 1e-5
TOL = 1e-3


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


def _torch_rms(h, w, eps):
    hf = h.float()
    rstd = torch.rsqrt(hf.pow(2).mean(-1, keepdim=True) + eps)
    return ((hf * rstd).to(h.dtype) * w)


def _torch_silu_mul(y):
    k = y.shape[-1] // 2
    g = y[..., :k].float()
    return (g / (1.0 + torch.exp(-g))).to(y.dtype) * y[..., k:]


def _block(seed):
    T = torch.bfloat16
    ks = {"o": (H, [H]), "gate_up": (H, [I, I]), "down": (I, [H]), "qkv": (H, QKV)}
    ks = {n: ParoLinearKernel.from_buffers(make_synthetic_layer(K, p, seed=seed + i, device="cuda"), T, check_pairs=False)
          for i, (n, (K, p)) in enumerate(ks.items())}
    g = torch.Generator().manual_seed(seed)
    w1 = (1.0 + 0.1 * torch.randn(H, generator=g)).to(T).cuda()
    w2 = (1.0 + 0.1 * torch.randn(H, generator=g)).to(T).cuda()
    return ks, w1, w2


class Unfused:
    """The same tail as single linears + torch element-wise ops, into fixed buffers."""

    def __init__(self, ks, w1, w2, attn, resid):
        self.ks, self.w1, self.w2, self.attn, self.resid = ks, w1, w2, attn, resid
        m, dt = attn.shape[0], attn.dtype
        self.o = torch.empty(m, H, dtype=dt, device="cuda")
        self.d = torch.empty(m, H, dtype=dt, device="cuda")
        self.bufs = {"residual_mid": torch.empty(m, H, dtype=dt, device="cuda"), "mlp_act": torch.empty(m, 2 * I, dtype=dt, device="cuda"),
                     "residual_out": torch.empty(m, H, dtype=dt, device="cuda"), "qkv": torch.empty(m, sum(QKV), dtype=dt, device="cuda")}

    def __call__(self):
        b, ks = self.bufs, self.ks
        ks["o"].forward_into(self.attn, self.o)
        torch.add(self.o, self.resid, out=b["residual_mid"])   # T(fp32 sum), as (o.float() + resid.float()).to(T)
        ks["gate_up"].forward_into(_torch_rms(b["residual_mid"], self.w1, EPS), b["mlp_act"])
        ks["down"].forward_into(_torch_silu_mul(b["mlp_act"]), self.d)
        torch.add(self.d, b["residual_mid"], out=b["residual_out"])
        ks["qkv"].forward_into(_torch_rms(b["residual_out"], self.w2, EPS), b["qkv"])


def _capture(fn):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        fn()
    torch.cuda.synchronize()
    return gr


def _launches(fn):
    from torch.profiler import ProfilerActivity, profile

    try:
        for _ in range(2):   # the first profiled call of a process can miss its first kernel: count the second
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                fn()
                torch.cuda.synchronize()
        return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "memcpy" not in e.name.lower()
                   and "memset" not in e.name.lower())
    except Exception as e:   # report, do not fail the measurement
        return f"not measured ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--sets", type=int, default=2)
    ap.add_argument("--M", default="32,64,128,256,1024,4096")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prefill_chain_bench needs a CUDA device")
    print(json.dumps({"gpu_before": _gpu()}), flush=True)
    blocks = [_block(100 * s + 1) for s in range(a.sets)]
    flops_per_row = 2 * (H * H + H * 2 * I + I * H + H * sum(QKV))
    ok = True
    for M in (int(m) for m in a.M.split(",")):
        g = torch.Generator(device="cuda").manual_seed(M)
        attn = torch.randn(M, H, generator=g, device="cuda").to(torch.bfloat16)
        resid = torch.randn(M, H, generator=g, device="cuda").to(torch.bfloat16)
        fused, unfused = [], []
        for ks, w1, w2 in blocks:
            ch, bufs = chain.decoder_tail(ks["o"], ks["gate_up"], ks["down"], ks["qkv"], attn_out=attn, residual=resid, post_attn_norm=w1,
                                          next_input_norm=w2, eps=EPS)
            fused.append((ch, bufs))
            unfused.append(Unfused(ks, w1, w2, attn, resid))
        # outputs of both variants on set 0, and the launches of one block
        fused[0][0]()
        n_fused = _cabi.last_launch_count()
        unfused[0]()
        torch.cuda.synchronize()
        errs = {n: float((fused[0][1][n].double() - b.double()).norm() / b.double().norm()) for n, b in unfused[0].bufs.items()}
        ok = ok and all(e <= TOL for e in errs.values())
        launches = {"prefill_chain": n_fused, "prefill_chain_profiler": _launches(fused[0][0]), "unfused_profiler": _launches(unfused[0])}
        graphs = [(_capture(ch), _capture(u)) for (ch, _), u in zip(fused, unfused)]
        for gf, gu in graphs:   # warm both graphs once more outside the timing
            gf.replay()
            gu.replay()
        torch.cuda.synchronize()
        ft, ut = [], []
        for it in range(a.iters):
            gf, gu = graphs[it % a.sets]
            e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
            if (it // a.sets) % 2:   # alternate which variant runs first, on every weight set
                e0.record(); gu.replay(); e1.record(); gf.replay(); e2.record()   # noqa: E702
                torch.cuda.synchronize()
                ut.append(e0.elapsed_time(e1) * 1e3); ft.append(e1.elapsed_time(e2) * 1e3)   # noqa: E702
            else:
                e0.record(); gf.replay(); e1.record(); gu.replay(); e2.record()   # noqa: E702
                torch.cuda.synchronize()
                ft.append(e0.elapsed_time(e1) * 1e3); ut.append(e1.elapsed_time(e2) * 1e3)   # noqa: E702
        tf, tu = _pct(ft, 0.5), _pct(ut, 0.5)
        print(json.dumps({
            "M": M, "prefill_chain_us": round(tf, 1), "chain_p25_p75": [round(_pct(ft, 0.25), 1), round(_pct(ft, 0.75), 1)],
            "unfused_us": round(tu, 1), "unfused_p25_p75": [round(_pct(ut, 0.25), 1), round(_pct(ut, 0.75), 1)],
            "speedup": round(tu / tf, 3), "chain_tflops": round(flops_per_row * M / tf / 1e6, 1),
            "unfused_tflops": round(flops_per_row * M / tu / 1e6, 1), "launches_per_block": launches,
            "rel_err_vs_unfused": {n: float(f"{e:.2e}") for n, e in errs.items()}}), flush=True)
        del fused, unfused, graphs
        torch.cuda.empty_cache()
    print(json.dumps({"gpu_after": _gpu(), "outputs_agree": ok}), flush=True)
    if not ok:
        raise SystemExit(f"the prefill chain and the unfused path disagree by more than {TOL}")


if __name__ == "__main__":
    main()
