#!/usr/bin/env python
"""bench.py -- the hot path of BASELINE.json: ParoQuant INT4 linears of Llama-3-8B.

  python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--m 1] [--dump-outputs DIR]

One "step" = one decode token through ALL quantised linears of Llama-3-8B (32 layers x
{merged qkv 4096->6144 (3 rotations), o 4096->4096, merged gate_up 4096->28672 (2 rotations),
down 14336->4096}) at batch M (default 1), bf16 activations, random-init weights in checkpoint
format, prepacked once.  Attention / norms / sampling are outside the hot path and are not run;
`value` is therefore decode tokens/s of the linear path, the part the reference's kernels own.
Per step 3.66 GB of packed weights are streamed (>> the H100's 50 MB L2), so no L2 flush is needed.

N > 1 (torchrun, one rank per GPU): the same model tensor-parallel -- qkv / gate_up column-sharded
(no communication), o / down row-sharded on 128-channel group boundaries + one NCCL all-reduce
each (strong scaling, as BASELINE.json config 5).

`--impl reference`: the reference's arithmetic on the host cores (oracle/cpu_baseline.py; the
reference itself is CUDA-only), a bounded sample per step.

`--dump-outputs DIR`: after the timed steps, what the timed paths computed in their last step is written as float32
DIR/<name>.npy (the inputs are seeded: the same arguments give the same inputs on every run).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import threading
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))

HIDDEN, KV, INTER = 4096, 1024, 14336
LAYERS = int(os.environ.get("BENCH_LAYERS", "32"))   # 32 = Llama-3-8B; smaller only for smoke-testing the harness
_VERBOSE = os.environ.get("BENCH_VERBOSE") == "1"


def _log(msg):
    if _VERBOSE:
        print(f"[bench r{os.environ.get('RANK', '0')}] {msg}", file=sys.stderr, flush=True)
SHAPES = {  # name: (K, part_sizes, kind)
    "qkv": (HIDDEN, [HIDDEN, KV, KV], "col"), "o": (HIDDEN, [HIDDEN], "row"),
    "gate_up": (HIDDEN, [INTER, INTER], "col"), "down": (INTER, [HIDDEN], "row"),
}


def measured_peaks():
    """HBM GB/s and dense bf16 TFLOP/s: MEASURED_PEAKS.json where the machine provides one, else the H100 SXM data sheet."""
    p = ROOT / "MEASURED_PEAKS.json"
    if p.exists():
        d = json.loads(p.read_text())
        return float(d["hbm_gbs"]), float(d.get("bf16_tflops", 989.0)), "measured"
    return 3350.0, 989.0, "h100_sxm_datasheet"


def algorithmic_bytes(K, parts, M, G=128, R=8):
    N, P = sum(parts), len(parts)
    return K * N // 2 + (K // G) * N * 2 + (K // G) * N // 2 + P * (R * K * 2 + R * (K // 2) * 2 + K * 2) + M * K * 2 + M * N * 2


class ClockSampler(threading.Thread):
    """SM clock + throttle reasons sampled in-process through NVML every few ms."""

    def __init__(self, index: int):
        super().__init__(daemon=True)
        self.samples, self.reasons, self.stop_flag, self.ok = [], set(), False, False
        try:
            import pynvml
            pynvml.nvmlInit()
            self.nv, self.h = pynvml, pynvml.nvmlDeviceGetHandleByIndex(index)
            self.max_mhz = pynvml.nvmlDeviceGetMaxClockInfo(self.h, pynvml.NVML_CLOCK_SM)
            self.ok = True
        except Exception:
            self.max_mhz = None

    def run(self):
        if not self.ok:
            return
        nv = self.nv
        names = {"hw_slowdown": nv.nvmlClocksEventReasonHwSlowdown, "hw_thermal_slowdown": nv.nvmlClocksEventReasonHwThermalSlowdown,
                 "sw_thermal_slowdown": nv.nvmlClocksEventReasonSwThermalSlowdown, "sw_power_cap": nv.nvmlClocksEventReasonSwPowerCap}
        while not self.stop_flag:
            try:
                self.samples.append(nv.nvmlDeviceGetClockInfo(self.h, nv.NVML_CLOCK_SM))
                r = nv.nvmlDeviceGetCurrentClocksEventReasons(self.h)
                self.reasons.update(k for k, bit in names.items() if r & bit)
            except Exception:
                pass
            time.sleep(0.004)

    def summary(self):
        if not self.samples:
            return {"sm_mhz": None, "sm_max_mhz": self.max_mhz, "reasons": ["unsampled"]}
        return {"sm_mhz": statistics.median(self.samples), "sm_max_mhz": self.max_mhz, "reasons": sorted(self.reasons), "samples": len(self.samples)}


# ------------------------------------------------------------------------------------------ ours
class DecodeModel:
    """All quantised linears of Llama-3-8B for one decode token at batch M, activations chained through the block:
    qkv -> [attention: not ours, stood in for by the q slice] -> o -> +residual, RMSNorm -> gate_up -> SiLU*up -> down
    -> +residual, RMSNorm -> next block's qkv.

    `token_chain`  1 + LAYERS launches: the first qkv, then per block ONE paro_chain_forward launch (o, gate_up, down and the
                   next block's qkv with the norms / activation / residual adds folded in) -- public API paroquant_b200.chain.
    `token_linear` 4 x LAYERS launches through the reference's operator surface, ParoLinearKernel.__call__ ==
                   torch.ops.paro.linear (what ParoQuantLinearMethod.apply calls); the element-wise neighbours are vLLM's
                   kernels there and are NOT run, so this is the lower bound of the unfused path."""

    def __init__(self, dev, M, dt, world=1, rank=0):
        import torch

        from paroquant_b200 import chain
        from paroquant_b200.checkpoint import make_synthetic_activations, make_synthetic_layer
        from paroquant_b200.linear import ParoLinearKernel

        self.torch, self.M, self.dev, self.world = torch, M, dev, world
        self.layers = []
        for li in range(LAYERS):
            lk = {}
            for si, name in enumerate(SHAPES):
                K, parts = shard_shape(name, world)
                buf = make_synthetic_layer(K, parts, seed=1234 + 16 * li + si + 1000 * rank, device=dev)
                lk[name] = ParoLinearKernel.from_buffers(buf, dt, check_pairs=(li == 0), max_m=max(M, 1))
                del buf
            self.layers.append(lk)
        torch.cuda.synchronize()
        self.x0 = make_synthetic_activations(M, HIDDEN, seed=77, device=dev, dtype=dt)
        self.x_host = make_synthetic_activations(M, HIDDEN, seed=77, dtype=dt).pin_memory()
        self.y_host = torch.empty(M, HIDDEN, dtype=dt).pin_memory()
        self.launches = 0
        self.chained = world == 1 or os.environ.get("BENCH_TP_NCCL") != "1"
        if self.chained:
            self.qkv0 = torch.empty(M, (HIDDEN + 2 * KV) // world, dtype=dt, device=dev)
            res = make_synthetic_activations(M, HIDDEN, seed=78, device=dev, dtype=dt)
            w = torch.ones(HIDDEN, dtype=dt, device=dev)
            self.res0, self.norm_w = res, w
            self.chains, self.copies = [], []
            qkv = self.qkv0
            for li, lk in enumerate(self.layers):
                hq = HIDDEN // world              # this rank's q columns of the (column-sharded) qkv output = o_proj's K shard
                if M == 1:
                    attn = qkv[:, :hq]                # the q slice of a single row is contiguous: no copy
                else:
                    attn = torch.empty(M, hq, dtype=dt, device=dev)
                    self.copies.append((attn, qkv))
                nxt = self.layers[li + 1]["qkv"] if li + 1 < LAYERS else None
                ch, bufs = chain.decoder_tail(lk["o"], lk["gate_up"], lk["down"], nxt, attn_out=attn, residual=res,
                                              post_attn_norm=w, next_input_norm=w if nxt is not None else None,
                                              tensor_parallel=world > 1)
                self.chains.append(ch)
                qkv, res = bufs["qkv"], bufs["residual_out"]
            self.final = res

    def token_chain(self):
        from paroquant_b200 import _cabi
        n = 0
        self.layers[0]["qkv"].forward_into(self.x0, self.qkv0)
        n += _cabi.last_launch_count()
        for li, ch in enumerate(self.chains):
            if self.M > 1:
                attn, qkv = self.copies[li]
                attn.copy_(qkv[:, :attn.shape[1]])       # a torch kernel, not counted as ours
            ch()
            n += _cabi.last_launch_count()
        self.launches = n
        return self.final

    def token_linear_with_neighbours(self):
        """token_linear + what vLLM launches between the linears (fused_add_rms_norm x2, silu_and_mul per block), as plain torch
        kernels: the same work a chain launch does -- the like-for-like partner of `token_chain`."""
        import torch.nn.functional as F
        from paroquant_b200 import _cabi
        n, x, res = 0, self.x0, self.res0
        w = self.norm_w
        for lk in self.layers:
            qkv = lk["qkv"](x); n += _cabi.last_launch_count()
            o = lk["o"](qkv[:, :HIDDEN]); n += _cabi.last_launch_count()
            res = o + res
            gu = lk["gate_up"](F.rms_norm(res, (HIDDEN,), w, 1e-5)); n += _cabi.last_launch_count()
            act = F.silu(gu[:, :INTER]) * gu[:, INTER:]
            d = lk["down"](act); n += _cabi.last_launch_count()
            res = d + res
            x = F.rms_norm(res, (HIDDEN,), w, 1e-5)
        self.launches = n
        return res

    def token_linear(self):
        from paroquant_b200 import _cabi
        n, x = 0, self.x0
        for lk in self.layers:
            qkv = lk["qkv"](x); n += _cabi.last_launch_count()
            o = lk["o"](qkv[:, :HIDDEN]); n += _cabi.last_launch_count()
            gu = lk["gate_up"](o); n += _cabi.last_launch_count()
            x = lk["down"](gu[:, :INTER]); n += _cabi.last_launch_count()
        self.launches = n
        return x


def shard_shape(name, world):
    K, parts, kind = SHAPES[name]
    if kind == "col":
        return K, [p // world for p in parts]
    return K // world, parts


def timed_graph(torch, fn, steps, warmup, barrier, use_graph=True):
    """Capture fn() as a CUDA graph (PDL edges included), W untimed replays, then K timed ones between CUDA events."""
    dev = torch.cuda.current_device()
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            out = fn()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    if use_graph:
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = fn()
        run = graph.replay
    else:
        run = fn
    for _ in range(max(warmup, 3)):
        run()
    barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        run()
    e1.record()
    barrier()
    return e0.elapsed_time(e1) / steps, run, out


def run_ours(args):
    import torch
    import torch.distributed as dist

    from paroquant_b200 import _cabi

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world != args.gpus:
        if args.gpus != 1:
            raise SystemExit(f"--gpus {args.gpus} needs torchrun with WORLD_SIZE={args.gpus} (got {world})")
        world, rank, local = 1, 0, 0
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
        _log("process group up")
    M = args.m
    dt = torch.bfloat16
    model = DecodeModel(dev, M, dt, world, rank)
    _log("weights prepacked")

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    use_graph = not args.no_graph
    if model.chained:
        # world > 1: the same chains on this rank's shards (qkv / gate_up column-sharded, o / down row-sharded on 128-channel
        # boundaries); the two all-reduces of a block happen INSIDE the chain launch (peer-memory block sums over NVLink)
        token = model.token_chain
    else:
        # tensor parallel: qkv / gate_up column-sharded, o / down row-sharded + all-reduce of the [M, 4096] partials
        xs = {name: torch.randn(M, shard_shape(name, world)[0], device=dev).to(dt) for name in SHAPES}
        outs = {name: torch.empty(M, sum(shard_shape(name, world)[1]), dtype=dt, device=dev) for name in SHAPES}

        def token():
            n = 0
            for lk in model.layers:
                for name in SHAPES:
                    lk[name].forward_into(xs[name], outs[name])
                    n += _cabi.last_launch_count()
                    if SHAPES[name][2] == "row":
                        dist.all_reduce(outs[name])
            model.launches = n
            return outs["down"]
        model.x0, model.final = xs["qkv"], outs["down"]

    sampler = ClockSampler(local)
    sampler.start()
    ms, run_step, final = timed_graph(torch, token, args.steps, args.warmup, barrier, use_graph)
    launches_per_step = model.launches
    dumps = {}
    if args.dump_outputs:   # the timed path's result of its last step, before anything else runs on these buffers
        dumps["chain_residual_out" if model.chained else "tp_down_out"] = final.float().cpu().numpy()
    _log(f"timed region done: {ms:.3f} ms/step")
    t_end = time.time() + 0.6   # keep the identical load running briefly so the NVML sampler sees clocks under this workload
    while time.time() < t_end:
        run_step()
        torch.cuda.synchronize()
    sampler.stop_flag = True
    sampler.join()

    # ---- end to end through the same public calls: host buffers in, host result out, every token (what a decode loop does)
    def e2e_step():
        model.x0.copy_(model.x_host, non_blocking=True)
        run_step()
        model.y_host.copy_(final, non_blocking=True)
        torch.cuda.current_stream().synchronize()   # the host consumes the result before the next token

    for _ in range(3):
        e2e_step()
    barrier()
    f0, f1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    f0.record()
    for _ in range(args.steps):
        e2e_step()
    f1.record()
    barrier()
    ms_e2e = f0.elapsed_time(f1) / args.steps

    per_linear = None
    chain_launches = launches_per_step
    if world == 1 and not args.no_per_linear:
        ms_l, run_l, final_l = timed_graph(torch, model.token_linear, args.steps, args.warmup, barrier, use_graph)
        if args.dump_outputs:
            dumps["per_linear_down_out"] = final_l.float().cpu().numpy()
        per_linear = {"tokens_per_s": M * 1e3 / ms_l, "ms_per_step": ms_l, "launches_per_step": model.launches,
                      "api": "ParoLinearKernel.__call__ -> torch.ops.paro.linear (the call ParoQuantLinearMethod.apply makes), one launch per "
                             "linear, activations chained by slices, vLLM's norm / activation kernels not run"}

    if per_linear is not None:
        ms_n, _, _ = timed_graph(torch, model.token_linear_with_neighbours, args.steps, args.warmup, barrier, use_graph)
        per_linear["with_neighbour_kernels"] = {"tokens_per_s": M * 1e3 / ms_n, "ms_per_step": ms_n,
                                                 "what": "the same 128 launches + torch's rms_norm / silu*mul / residual-add kernels between them: "
                                                         "the work one chain launch per block does"}
    chain_res = {"tokens_per_s": M * 1e3 / ms, "ms_per_step": ms, "launches_per_step": chain_launches, "e2e_tokens_per_s": M * 1e3 / ms_e2e,
                 "api": "paroquant_b200.chain.ParoChain (paro_chain_forward): norms, SiLU*up and residual adds folded in"}
    headline = "chain"
    if per_linear is not None and per_linear["ms_per_step"] < ms:
        # the per-linear operator surface is the faster public path on this run: it is the headline, measured end to end the same way
        headline = "per_linear"

        def e2e_step_l():
            model.x0.copy_(model.x_host, non_blocking=True)
            run_l()
            model.y_host.copy_(final_l, non_blocking=True)
            torch.cuda.current_stream().synchronize()

        for _ in range(3):
            e2e_step_l()
        barrier()
        f0.record()
        for _ in range(args.steps):
            e2e_step_l()
        f1.record()
        barrier()
        ms_e2e = f0.elapsed_time(f1) / args.steps
        per_linear["e2e_tokens_per_s"] = M * 1e3 / ms_e2e
        ms, launches_per_step = per_linear["ms_per_step"], per_linear["launches_per_step"]

    if world > 1:
        t = torch.tensor([ms, ms_e2e], device=dev, dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms, ms_e2e = t.tolist()

    if rank == 0:
        hbm_peak, _, src = measured_peaks()
        step_bytes = LAYERS * sum(algorithmic_bytes(*shard_shape(n, world), M) for n in SHAPES)      # per rank
        achieved = step_bytes / (ms * 1e-3) / 1e9
        path = ("1 + %d launches: first qkv, then per block ONE chain launch (o -> +res/RMSNorm -> gate_up -> SiLU*up -> down -> "
                "+res/RMSNorm -> next qkv)" % LAYERS) if model.chained else "one launch per linear + NCCL all-reduce after o / down"
        if model.chained and world > 1:
            path += "; o / down row-sharded, their all-reduce fused into the launch (block sums written to every rank's peer buffer over NVLink)"
        line = {
            "metric": "llama3_8b_int4_decode_tokens_per_s", "value": M * 1e3 / ms, "unit": "tokens/s", "n_gpus": world,
            "steps": args.steps, "warmup": max(args.warmup, 3), "ms_per_step": ms, "higher_is_better": True,
            "scaling": "strong", "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
            "config": {"workload": f"Llama-3-8B all quantised linears, decode batch {M}: {LAYERS} x (qkv 4096->6144 P=3, o 4096->4096, "
                                   f"gate_up 4096->28672 P=2, down 14336->4096), INT4 g128 krot8, fused rotate+dequant+GEMV, activations chained",
                       "batch": M, "parallelism": f"tp{world}", "launch": "cuda_graph+pdl" if use_graph else "eager+pdl", "path": path,
                       "l2": "3.66 GB of weights streamed per step >> 50 MB L2, no flush needed"},
            "e2e": {"value": M * 1e3 / ms_e2e, "unit": "tokens/s", "h2d_bytes_per_step": model.x_host.numel() * 2, "d2h_bytes_per_step": model.y_host.numel() * 2,
                    "api": "paroquant_b200.chain.ParoChain.__call__ + ParoLinearKernel.forward_into" if model.chained else "ParoLinearKernel.forward_into + dist.all_reduce"},
            "gpu_launches": launches_per_step * args.steps,
            "clocks": sampler.summary(),
            "roofline": {"bound": "hbm", "achieved": achieved, "peak": hbm_peak, "unit": "GB/s", "frac": achieved / hbm_peak,
                         "peak_source": src, "kernel": "paro::stream_kernel", "launches_per_step": launches_per_step,
                         "algorithmic_bytes_per_step": step_bytes, "avg_launch_us": ms * 1e3 / max(launches_per_step, 1)},
        }
        line["config"]["headline_path"] = headline
        if world == 1:
            chain_res["frac_hbm"] = step_bytes / (chain_res["ms_per_step"] * 1e-3) / 1e9 / hbm_peak
            line["chain"] = chain_res
        if per_linear is not None:
            per_linear["frac_hbm"] = step_bytes / (per_linear["ms_per_step"] * 1e-3) / 1e9 / hbm_peak
            line["per_linear"] = per_linear
        if headline == "per_linear":
            line["config"]["path"] = "128 launches, one per (merged) linear, through torch.ops.paro.linear; activations chained by slices"
            line["e2e"]["api"] = "ParoLinearKernel.__call__ -> torch.ops.paro.linear"
            line["roofline"]["kernel"] = "paro::decode_kernel"
        if world == 1 and not args.no_ref_gpu:
            line["vs_reference_gpu"] = reference_gpu_section(M, line["value"], per_linear)
        if world == 1 and not args.no_prefill:
            line["prefill"] = prefill_section(dev)
            line["decode_batches"] = decode_batches_section(dev)
        if world == 1 and not args.no_prefill:
            try:
                line["training_op"] = training_op_section()
            except Exception as e:   # a side measurement must never cost the bench line
                line["training_op"] = {"unavailable": repr(e)[:200]}
        if world == 1 and not args.no_cpu_baseline:
            line["cpu_baseline"] = cpu_baseline_sample(M)
        if args.dump_outputs:
            import numpy as np
            out_dir = Path(args.dump_outputs)
            out_dir.mkdir(parents=True, exist_ok=True)
            for name, arr in dumps.items():
                np.save(out_dir / f"{name}.npy", arr)
        print(json.dumps(line), flush=True)
    if world > 1:
        # destroy_process_group() can block for minutes in the NCCL heartbeat monitor once torchrun's TCPStore
        # goes away (seen on the 2-GPU box: all work done, processes never exit).  Everything is flushed: leave.
        dist.barrier()
        torch.cuda.synchronize()
        sys.stdout.flush()
        sys.stderr.flush()
        os._exit(0)


def reference_gpu_section(M, ours_tok_s, per_linear):
    """BASELINE config 4, "vs reference paroquant/kernels on same box": the UNMODIFIED reference pair (its rotate kernel from
    oracle/_ref + vLLM's AWQ-Marlin, per partition, + cat: plugin.py:288-311) timed like for like in a SEPARATE process
    (tools/ref_gpu.py bench: same shapes, weight sets > L2, one CUDA graph, CUDA events).  A reported baseline."""
    import subprocess
    import tempfile

    so = ROOT / "oracle" / "_ref" / "paroquant_rotation.so"
    if not so.exists():
        return {"unavailable": "oracle/_ref/paroquant_rotation.so not built (needs /root/reference at build time)"}
    with tempfile.TemporaryDirectory() as d:
        out = Path(d) / "ref.json"
        try:
            r = subprocess.run([sys.executable, str(ROOT / "tools" / "ref_gpu.py"), "bench", str(out), "--m", f"{M},4096"],
                               capture_output=True, text=True, timeout=900)
        except subprocess.TimeoutExpired:
            return {"unavailable": "tools/ref_gpu.py bench timed out"}
        if r.returncode or not out.exists():
            return {"unavailable": (r.stderr or r.stdout)[-300:]}
        res = json.loads(out.read_text())
    per = {k: v["us_per_linear"] for k, v in res.items() if v["M"] == M}
    us_layer = sum(per[f"{n}_m{M}"] for n in SHAPES)
    tok_s = M * 1e6 / (LAYERS * us_layer)
    sec = {"tokens_per_s": tok_s, "us_per_layer": us_layer, "per_linear_us": per, "ratio": ours_tok_s / tok_s,
           "what": "reference rotate (oracle/_ref) + vLLM 0.22 AWQ-Marlin per partition + cat, linears only, CUDA graph, same box",
           "prefill_4096_tflops": {k: v["tflops"] for k, v in res.items() if v["M"] == 4096}}
    if per_linear is not None:
        sec["ratio_per_linear_api"] = per_linear["tokens_per_s"] / tok_s
    return sec


def training_op_section():
    """SURVEY 8(f) rank 4: the rotate op's backward on fp32 [4096, 4096] (the optimiser's dtype), ONE launch (paro_rotate_backward)
    against the reference's backward structure -- a Python walk over the 8 rotations with per-rotation launches, gathers and
    reductions (kernels/cuda/autograd.py:20-61) -- run on our own rotate kernel on the same box (tools/backward_bench.py)."""
    import torch

    import paroquant_b200.kernels.cuda  # noqa: F401
    from paroquant_b200 import _cabi
    from paroquant_b200.checkpoint import make_synthetic_layer
    from tools.backward_bench import stagewise, timed

    M, K, G = 4096, 4096, 128
    L = make_synthetic_layer(K, [64], seed=5, device="cuda")
    pr, th, sc = L.pairs[0], L.theta[0].float(), L.channel_scales[0].float().view(-1)
    x = torch.randn(M, K, device="cuda")
    go = torch.randn(M, K, device="cuda")
    y = torch.ops.rotation.rotate(x, pr, th, sc, G)
    fwd = timed(lambda: torch.ops.rotation.rotate(x, pr, th, sc, G))
    fused = timed(lambda: _cabi.rotate_backward(y, go, x, pr, th, sc, G))
    walk = timed(lambda: stagewise(x, pr, th, y, go, sc, G), reps=5)
    return {"shape": [M, K], "dtype": "f32", "krot": 8, "forward_us": fwd, "fused_backward_us": fused, "stagewise_walk_us": walk,
            "speedup_vs_walk": walk / fused, "fused_backward_GBps": 4 * M * K * 4 / fused / 1e3}


def prefill_section(dev):
    """BASELINE.json config 3 beside the decode headline: fused rotate + dequant + wgmma GEMM at batch 256 / 1024 / 4096 on the
    Llama-3-8B linear shapes plus the K = 11008 down projection, TFLOP/s against the measured bf16 tensor roofline (each call:
    rotation pre-pass + GEMM).  The headline figure is the 4096-token layer."""
    import torch

    from paroquant_b200.checkpoint import make_synthetic_activations, make_synthetic_layer
    from paroquant_b200.linear import ParoLinearKernel

    _, tf_peak, src = measured_peaks()
    shapes = {n: (K, parts) for n, (K, parts, _) in SHAPES.items()}
    shapes["llama2_down"] = (11008, [HIDDEN])
    cells, out4096, tot_fl, tot_us = {}, {}, 0.0, 0.0
    for name, (K, parts) in shapes.items():
        k = ParoLinearKernel.from_buffers(make_synthetic_layer(K, parts, seed=99, device=dev), torch.bfloat16, check_pairs=False, max_m=4096)
        for Mp in (256, 1024, 4096):
            x = make_synthetic_activations(Mp, K, seed=5, device=dev)
            y = torch.empty(Mp, sum(parts), dtype=torch.bfloat16, device=dev)
            for _ in range(3):
                k.forward_into(x, y)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            reps = 10
            e0.record()
            for _ in range(reps):
                k.forward_into(x, y)
            e1.record()
            torch.cuda.synchronize()
            us = e0.elapsed_time(e1) * 1e3 / reps
            fl = 2.0 * Mp * K * sum(parts)
            cells[f"{name}_m{Mp}"] = {"us": us, "tflops": fl / us / 1e6, "frac_tensor": fl / us / 1e6 / tf_peak}
            if Mp == 4096 and name in SHAPES:
                out4096[name] = {"us": us, "tflops": fl / us / 1e6}
                tot_fl += fl
                tot_us += us
            del x, y
        del k
        torch.cuda.empty_cache()
    return {"batch": 4096, "tflops": tot_fl / tot_us / 1e6, "frac_tensor": tot_fl / tot_us / 1e6 / tf_peak, "peak_tflops": tf_peak,
            "peak_source": src, "per_linear": out4096, "cells": cells,
            "note": "headline: one Llama-3-8B layer's quantised linears at 4096 tokens, rotation pre-pass included; cells: every shape "
                    "(+ K = 11008) x batch 256 / 1024 / 4096"}


def decode_batches_section(dev):
    """BASELINE.json config 2: the fused rotate + dequant + GEMV per shape at batch 1 / 4 / 16 (weight sets > L2 cycled, one CUDA
    graph, PDL edges), HBM GB/s against the measured roofline."""
    import torch

    from paroquant_b200.checkpoint import make_synthetic_activations, make_synthetic_layer
    from paroquant_b200.linear import ParoLinearKernel

    hbm_peak, _, _ = measured_peaks()
    out = {}
    for name, (K, parts, _) in SHAPES.items():
        nsets = max(3, int(300e6 // (K * sum(parts) // 2)) + 1)
        ks = [ParoLinearKernel.from_buffers(make_synthetic_layer(K, parts, seed=900 + i, device=dev), torch.bfloat16, check_pairs=False)
              for i in range(nsets)]
        for M in (1, 4, 16):
            x = make_synthetic_activations(M, K, seed=1, device=dev)
            y = torch.empty(M, sum(parts), dtype=torch.bfloat16, device=dev)

            def sweep():
                for k in ks:
                    k.forward_into(x, y)

            ms, _, _ = timed_graph(torch, sweep, 10, 3, torch.cuda.synchronize)
            us = ms * 1e3 / nsets
            ab = algorithmic_bytes(K, parts, M)
            out[f"{name}_m{M}"] = {"us": us, "GBps": ab / us / 1e3, "frac_hbm": ab / us / 1e3 / hbm_peak}
        del ks
        torch.cuda.empty_cache()
    return out


# ------------------------------------------------------------------------------------------ CPU baseline / reference arm
CPU_SAMPLE = ["qkv", "o"]   # the attention-side linears of ONE layer: the same bounded sample in both arms


def cpu_sample_seconds(M, repeats=3):
    """Median seconds of `repeats` passes (after one warm-up pass) over the sample, all host threads, dequant on every call
    (the reference keeps INT4 weights and dequantises inside the GEMM; oracle/cpu_baseline.py is its arithmetic on torch CPU)."""
    import torch

    from oracle import cpu_baseline as cb
    from paroquant_b200.checkpoint import make_synthetic_activations, make_synthetic_layer

    threads = os.cpu_count() or 1
    torch.set_num_threads(threads)
    lay = [make_synthetic_layer(SHAPES[n][0], SHAPES[n][1], seed=1234 + i) for i, n in enumerate(CPU_SAMPLE)]
    xs = [make_synthetic_activations(M, SHAPES[n][0], seed=77 + i, dtype=torch.bfloat16) for i, n in enumerate(CPU_SAMPLE)]
    cb.time_sample(lay, xs)
    times = sorted(cb.time_sample(lay, xs) for _ in range(repeats))
    frac = sum(algorithmic_bytes(SHAPES[n][0], SHAPES[n][1], M) for n in CPU_SAMPLE) / sum(algorithmic_bytes(SHAPES[n][0], SHAPES[n][1], M) for n in SHAPES) / LAYERS
    return times[len(times) // 2], times, frac, threads


def cpu_baseline_sample(M):
    sec, times, frac, threads = cpu_sample_seconds(M)
    return {"value": M * frac / sec, "unit": "tokens/s", "cores": threads, "kind": "port",
            "sample": f"qkv + o of one layer = {frac:.5f} of a token's weight bytes, dequant+rotate+matmul per call on torch CPU, "
                      f"median of {len(times)} passes after a warm-up ({', '.join(f'{t:.2f}' for t in times)} s), scaled to tokens/s",
            "seconds_per_sample": sec}


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    M = args.m
    steps = max(3, min(args.steps, 5))
    sec, times, frac, threads = cpu_sample_seconds(M, repeats=steps)
    tok_s = M * frac / sec
    line = {"impl": "reference", "metric": "llama3_8b_int4_decode_tokens_per_s", "value": tok_s, "unit": "tokens/s",
            "n_gpus": args.gpus, "steps": steps, "warmup": 1, "ms_per_step": sec * 1e3, "higher_is_better": True,
            "scaling": "strong", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": {"workload": f"Llama-3-8B all quantised linears, decode batch {M} (CPU port of the reference math; the reference has no CPU path)",
                       "batch": M, "parallelism": "cpu"},
            "cpu_baseline": {"value": tok_s, "unit": "tokens/s", "cores": threads, "kind": "port",
                             "sample": f"per step: qkv + o of one layer = {frac:.5f} of a token's weight bytes, dequant+rotate+matmul, median of {steps} "
                                       f"passes after a warm-up, scaled to tokens/s"},
            "e2e": {"value": tok_s, "unit": "tokens/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--m", type=int, default=1, help="decode batch (rows per linear), 1..16")
    ap.add_argument("--no-graph", action="store_true")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-prefill", action="store_true")
    ap.add_argument("--no-ref-gpu", action="store_true")
    ap.add_argument("--no-per-linear", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", help="write the timed paths' outputs of their last step as DIR/<name>.npy")
    args = ap.parse_args()
    if args.impl == "reference":
        run_reference(args)
    else:
        run_ours(args)


if __name__ == "__main__":
    main()
