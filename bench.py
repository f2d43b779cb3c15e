"""bench.py — denoiser steps/sec of the Stage-I temporal-3D-diffusion hot path (BASELINE.json metric) on N H100s.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl reference] [--mode temporal|dp] [--dump-outputs DIR]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P bench.py --gpus N ...

One "step" = one denoiser step of the default window (SURVEY 8(d), config c2): CFG batch of 2 branches x T=16 frames x
N=2048 latent tokens (+1 time token) through the 21-block DiT (width 2048, 16 heads), CFG combine (7.5) + Euler update.
5.469e14 algorithmic FLOP per step, of which the inflated self-attention QK^T+PV is 3.698e14 (BASELINE.md section 2).
Weights are seeded-random (no checkpoints offline), inputs synthetic; the per-step working set (2.9 GB weights +
GBs of activations) is far larger than the 50 MB L2, so no explicit L2 flush is needed between iterations.

Prints ONE JSON line (rank 0).
  N = 1: `value` = steps/s of the window on one GPU.
  N > 1: `value` = steps/s of ONE window whose 16 frames are sharded over the N ranks, the temporal-attention K/V
         all-gathered per layer over NVLink (`--mode temporal`, the default: STRONG scaling, the only path with a collective
         on it — BASELINE config 5's window).  `--mode dp` makes the whole-clip data-parallel aggregate (one independent
         window per GPU, no collective, weak scaling — BASELINE config 4) the headline instead; either way the other figure
         is reported under `dp` / `temporal_shard`.
`--impl reference` times the reference's own CPU path (the fp32 oracle port, all host threads) on a fixed bounded sample.
`--dump-outputs DIR` writes, after the timed steps, the denoised latents of the timed window (what `denoise()` returns to
its caller, (1, 16, 2048, 64) float32) as DIR/latents.npy.  Weights and inputs are seeded, so two builds run with the same
arguments can be compared output for output.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

F_STEP = 5.469e14          # algorithmic FLOP per denoiser step, T=16 (BASELINE.md section 2)
F_ATTN_LAUNCH = 4.0 * 2 * (16 * 2049) ** 2 * 2048   # one inflated self-attention launch (QK^T + PV), B=2
METRIC = "denoiser_steps_per_sec"
UNIT = "steps/s"
WORKLOAD = "davis_camel-shaped default window: CFG x2, T=16 frames, N=2048 tokens, 21-block DiT width 2048, guidance 7.5"
ATTN_KERNEL = "flash_attn_fwd_kernel<128> (inflated self-attention, d_h 128, wgmma)"
T_WIN, N_TOK, C_LAT, S_CTX, D_CTX = 16, 2048, 64, 257, 1024
CPU_SAMPLE_T = 8           # frames of the fixed CPU sample (identical in every run: BENCH, SCALE, --impl reference)


def _peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return d.get("bf16_tflops_sustained", NOMINAL_BF16_TF), d.get("hbm_gbs", NOMINAL_HBM_GBS), "measured (MEASURED_PEAKS.json: sustained bf16 / hbm_gbs)"
    return NOMINAL_BF16_TF, NOMINAL_HBM_GBS, "H100 SXM data sheet (dense bf16, HBM3), not a measured figure"


class ClockSampler:
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index: int):
        self.f = tempfile.NamedTemporaryFile("w+", suffix=".csv", delete=False)
        try:
            self.p = subprocess.Popen(["nvidia-smi", "-i", str(index), f"--query-gpu={self.Q}",
                                       "--format=csv,noheader,nounits", "-lms", "200"], stdout=self.f,
                                      stderr=subprocess.DEVNULL)
        except Exception:  # noqa: BLE001
            self.p = None

    def stop(self) -> dict:
        if self.p is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.p.terminate()
        try:
            self.p.wait(timeout=5)
        except Exception:  # noqa: BLE001
            self.p.kill()
        self.f.flush()
        rows = [l.strip().split(", ") for l in open(self.f.name) if l.strip()]
        os.unlink(self.f.name)
        sm = sorted(int(float(r[0])) for r in rows if len(r) >= 7)
        reasons = set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for r in rows:
            if len(r) >= 7:
                for nme, v in zip(names, r[3:7]):
                    if v.strip().lower().startswith("active"):
                        reasons.add(nme)
        return {"sm_mhz": sm[len(sm) // 2] if sm else None,
                "sm_max_mhz": int(float(rows[0][1])) if rows and len(rows[0]) >= 2 else None,
                "power_w_max": max((float(r[2]) for r in rows if len(r) >= 7), default=None),
                "samples": len(sm), "reasons": sorted(reasons)}


# ------------------------------------------------------------------------------------------------ reference (CPU) arm
def cpu_reference_sample(threads: int, T: int = CPU_SAMPLE_T, N: int = N_TOK):
    """One DiT block (block.py:110-154) of the cond branch at T frames x (N+1) tokens through the fp32 oracle port.
    Returns (seconds, FLOPs of the sample)."""
    import torch

    from oracle import denoiser_oracle as do
    from oracle import synth

    torch.set_num_threads(threads)
    cfg = do.DenoiserConfig(num_layers=1, inflated_layers=(0,))
    if not hasattr(cpu_reference_sample, "_sd"):
        cpu_reference_sample._sd = {k: v for k, v in synth.make_state_dict(cfg, 1234).items()}
    sd = cpu_reference_sample._sd
    g = torch.Generator().manual_seed(0)
    L = N + 1
    h = torch.randn(T, L, cfg.width, generator=g)
    ctx = torch.randn(T, 257, cfg.cross_attention_dim, generator=g)
    pos = torch.arange(T, dtype=torch.float32)
    cos, sin = do.rotary_tables(cfg.head_dim, pos)
    rope = (cos[:, None].repeat(1, L, 1), sin[:, None].repeat(1, L, 1))
    t0 = time.perf_counter()
    with torch.no_grad():
        do.block_forward(sd, "blocks.0.", h, ctx, cfg.num_attention_heads, T, True, rope, None)
    dt = time.perf_counter() - t0
    S = T * L
    D, F_, Dc = cfg.width, int(cfg.width * cfg.mlp_ratio), cfg.cross_attention_dim
    flops = 4.0 * S * S * D + 4.0 * S * 257 * D + 2.0 * S * D * (6 * D + 2 * F_) + 2.0 * (T * 257) * Dc * 2 * D
    return dt, flops


def cpu_baseline(repeats: int, warmup: int = 1) -> dict:
    """The reference's CPU path on this box: the SAME fixed sample every time (T=8 frames of one block), one warm-up,
    `repeats` timed runs, MEDIAN; extrapolated by FLOPs to the 5.469e14-FLOP step."""
    threads = os.cpu_count() or 1
    for _ in range(warmup):
        cpu_reference_sample(threads)
    runs = [cpu_reference_sample(threads) for _ in range(max(1, repeats))]
    sec = statistics.median(r[0] for r in runs)
    fl = runs[0][1]
    rate = fl / sec
    sample = (f"1 of 21 DiT blocks, cond branch, T={CPU_SAMPLE_T} frames x 2049 tokens ({fl:.3e} FLOP), fp32 oracle port of the "
              f"reference modules (oracle/denoiser_oracle.py), median of {len(runs)} runs after {warmup} warm-up: {sec:.2f} s "
              f"= {rate / 1e12:.3f} TFLOP/s on {threads} threads, extrapolated by FLOPs to the {F_STEP:.3e}-FLOP step")
    return {"value": rate / F_STEP, "unit": UNIT, "cores": threads, "kind": "port", "sample": sample,
            "runs_s": [round(r[0], 3) for r in runs]}


def run_reference(args, rank: int):
    if rank != 0:
        return
    cpu = cpu_baseline(repeats=max(3, args.steps), warmup=max(1, min(args.warmup, 2)))
    v = cpu["value"]
    line = {
        "impl": "reference", "metric": METRIC, "value": v, "unit": UNIT, "n_gpus": args.gpus,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": 1000.0 / v, "higher_is_better": True,
        "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": WORKLOAD, "sample": cpu["sample"]},
        "cpu_baseline": cpu,
        "e2e": {"value": v, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }
    print(json.dumps(line), flush=True)


# ------------------------------------------------------------------------------------------------ reference recipe on the GPU
def gpu_eager_baseline(dev, steps: int = 3) -> dict:
    """The reference's own GPU recipe on the same GPU: the oracle restatement of the reference modules (same op sequence:
    nn.Linear-equivalent matmuls, F.layer_norm, RMSNorm, RoPE, F.scaled_dot_product_attention, GELU) in PyTorch eager under
    torch.autocast(bf16) (pipeline.py:671), cuBLAS + torch's SDPA backend, plus the CFG combine / Euler update in torch."""
    import torch

    from oracle import denoiser_oracle as do
    from oracle import synth

    cfg = do.DenoiserConfig()
    sd = synth.make_state_dict(cfg, 1234, device=dev)
    T, N = T_WIN, N_TOK
    g = torch.Generator(device=dev).manual_seed(1)
    lat = torch.randn(1, T, N, C_LAT, device=dev, generator=g)
    ctx = torch.randn(1, T, S_CTX, D_CTX, device=dev, generator=g)
    mask = torch.zeros(1, T, device=dev)
    mask[0, 0] = 1
    fs = torch.arange(T, dtype=torch.float32, device=dev)[None]

    def step(freqs):
        h, c, m, f = do.cfg_batch(lat, ctx, mask, fs, ((0, 1), (1, 1)))
        t = torch.tensor([500.0, 500.0], device=dev)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out, freqs = do.denoiser_forward(sd, cfg, h, c, f, t, m, freqs)
        v = do.cfg_aggregate(out, [7.5], 2)
        upd = lat + 0.01 * v
        lat[mask == 0] = upd[mask == 0].float()
        return freqs

    with torch.no_grad():
        fr = step(None)
        fr = step(fr)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fr = step(fr)
        e1.record()
        torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    del sd, fr
    torch.cuda.empty_cache()
    return {"value": 1000.0 / ms, "unit": UNIT, "ms_per_step": ms, "steps": steps,
            "what": "oracle restatement of the reference modules, PyTorch eager, autocast bf16, cuBLAS + torch SDPA, same GPU, "
                    f"same window shape (torch {torch.__version__})"}


# ------------------------------------------------------------------------------------------------ CUDA arm
def run_b200(args):
    import torch
    import torch.distributed as dist

    from actionmesh_b200 import ops
    from actionmesh_b200.denoiser import B200Denoiser, DenoiserConfig
    from actionmesh_b200.guidance import ClassifierFreeGuidance
    from actionmesh_b200.scheduler import B200SchedulerFlow

    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    shard = None
    if world > 1:
        from actionmesh_b200.window_shard import FrameShard, PeerFrameShard, configure_nccl_env

        configure_nccl_env()  # NCCL protocol / channel defaults for the sharded window's K/V all-gather (before init)
        dist.init_process_group("nccl", device_id=dev)
        if T_WIN % world == 0:
            if args.exchange == "peer" and not PeerFrameShard.available(dev):
                args.exchange = "nccl"  # no symmetric memory on this box: the NCCL all-gather is the other exchange
            shard = PeerFrameShard() if args.exchange == "peer" else FrameShard()
    K, W = args.steps, max(args.warmup, 0)
    T, N, C, S, Dc = T_WIN, N_TOK, C_LAT, S_CTX, D_CTX
    temporal_main = world > 1 and args.mode == "temporal" and shard is not None

    model = B200Denoiser(DenoiserConfig()).to(dev)
    model.init_random_(seed=1234)  # same seed on every rank => replicated weights
    cf = ClassifierFreeGuidance(guidance_at_inference=[[0, 1], [1, 1]], guidance_scales=[7.5])
    framestep = torch.arange(T, dtype=torch.float32)[None]
    host_mask = torch.zeros(1, T)
    host_mask[0, 0] = 1.0  # anchor frame observed, like the first AR window

    def host_inputs(seed_off: int):
        g = torch.Generator(device="cpu").manual_seed(44 + seed_off)
        lat = torch.randn(1, T, N, C, generator=g).pin_memory()
        ctx = torch.randn(1, T, S, Dc, generator=torch.Generator().manual_seed(5 + seed_off)).pin_memory()
        return lat, ctx

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def allmax(ms: float) -> float:
        t = torch.tensor([ms], device=dev, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    def timed_window(host_lat, host_ctx, use_shard, tags=None):
        """W + K steps of one denoise() call on device-resident inputs; CUDA events around the last K steps, max over ranks."""
        sch = B200SchedulerFlow(num_inference_steps=W + K, shift=3.0, is_additive=True)
        lat, ctx, mask = host_lat.to(dev), host_ctx.to(dev), host_mask.to(dev)
        ev, marks = {}, {"launch0": 0}

        def cb(step, total):
            if step == W:
                ev["t0"] = torch.cuda.Event(enable_timing=True)
                ev["t0"].record()
                marks["launch0"] = ops.launch_count
                if tags:
                    ops.event_log, ops.event_tags = [], set(tags)
            if step == total:
                ev["t1"] = torch.cuda.Event(enable_timing=True)
                ev["t1"].record()

        barrier()
        if W == 0:
            cb(0, W + K)
        sch.denoise(model, cf, lat, ctx, device=dev, mask=mask, framestep=framestep, step_callback=cb,
                    shard=shard if use_shard else None)
        barrier()
        log = ops.event_log
        ops.event_log = None
        return (allmax(ev["t0"].elapsed_time(ev["t1"])), ops.launch_count - marks["launch0"], log, ev["t0"].elapsed_time(ev["t1"]),
                lat)

    def timed_e2e(host_lat, host_ctx, use_shard):
        """The same metric through the public API with HOST buffers: inputs copied from pinned memory inside the timed region,
        the latents read back to the host after every step."""
        sch = B200SchedulerFlow(num_inference_steps=K, shift=3.0, is_additive=True)
        host_out = torch.empty(1, T, N, C).pin_memory()
        d2h = {"bytes": 0}
        holder = {}

        def cb(step, total):
            if not use_shard:  # (sharded: each rank's slice lives in a private buffer; the full window is read at the end)
                host_out.copy_(holder["x"], non_blocking=True)
                d2h["bytes"] += host_out.numel() * 4

        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        lat = host_lat.to(dev, non_blocking=True)
        ctx = host_ctx.to(dev, non_blocking=True)
        mask = host_mask.to(dev, non_blocking=True)
        holder["x"] = lat
        out = sch.denoise(model, cf, lat, ctx, device=dev, mask=mask, framestep=framestep, step_callback=cb,
                          shard=shard if use_shard else None)
        host_out.copy_(out, non_blocking=True)
        e1.record()
        barrier()
        ms = allmax(e0.elapsed_time(e1))
        h2d = (host_lat.numel() + host_ctx.numel() + host_mask.numel()) * 4
        return ms, h2d // K, (d2h["bytes"] + host_out.numel() * 4) // K

    # ---------------- headline (`value`) + end-to-end
    sampler = ClockSampler(local) if rank == 0 else None
    if temporal_main:
        hl, hc = host_inputs(0)                     # the SAME window on every rank
        ms_total, launches, log, ms_local, out = timed_window(hl, hc, True, tags={"attn_self"})  # (few host cycles to spare per launch here)
        value = K / (ms_total / 1e3)
        scaling = "strong"
        clocks = sampler.stop() if sampler else None
        e2e_ms, h2d, d2h = timed_e2e(hl, hc, True)
        e2e_val = K / (e2e_ms / 1e3)
    else:
        hl, hc = host_inputs(rank)                  # one independent window per GPU
        ms_total, launches, log, ms_local, out = timed_window(hl, hc, False, tags={"attn_self", "gemm", "layernorm"})
        value = world * K / (ms_total / 1e3)
        scaling = "weak"
        clocks = sampler.stop() if sampler else None
        e2e_ms, h2d, d2h = timed_e2e(hl, hc, False)
        e2e_val = world * K / (e2e_ms / 1e3)

    if args.dump_outputs and rank == 0:
        import numpy as np

        os.makedirs(args.dump_outputs, exist_ok=True)
        np.save(os.path.join(args.dump_outputs, "latents.npy"), out.detach().float().cpu().numpy())
    del out

    # ---------------- N > 1: the other multi-GPU figure
    other = None
    if world > 1:
        try:
            if temporal_main:
                hl2, hc2 = host_inputs(rank)
                ms2 = timed_window(hl2, hc2, False)[0]
                other = ("dp", {"value": world * K / (ms2 / 1e3), "unit": UNIT, "ms_per_step": ms2 / K, "scaling": "weak",
                                "note": "whole-clip data parallel: one independent window per GPU, no data-path collective"})
            elif shard is not None:
                hl2, hc2 = host_inputs(0)
                ms2 = timed_window(hl2, hc2, True)[0]
                other = ("temporal_shard", {"value": K / (ms2 / 1e3), "unit": UNIT, "ms_per_step": ms2 / K, "scaling": "strong",
                                            "frames_per_rank": T // world,
                                            "note": "ONE window, frames sharded over the ranks, temporal-attention K/V all-gathered per layer"})
        except Exception as exc:  # noqa: BLE001 - an optional leg must never cost the main JSON line
            other = ("other_mode", {"error": f"{type(exc).__name__}: {exc}"[:400]})

    # ---------------- sec/video of the Stage-I path through the public pipeline API (N = 1 only): 16 synthetic RGB frames
    # -> CUDA preprocessing (PIL-exact bicubic resize/crop/normalise) -> DinoV2-L -> one 16-frame window, default 30 steps, CFG 7.5; then Stage II (Stage 0 out of scope)
    video = None
    if world == 1 and not args.no_video:
        video = _video_leg(torch, ops, model, cf, dev)

    eager = None
    if world == 1 and not args.no_eager:
        try:
            torch.cuda.empty_cache()
            eager = gpu_eager_baseline(dev)
        except Exception as exc:  # noqa: BLE001
            eager = {"error": f"{type(exc).__name__}: {exc}"[:400]}

    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return
    peak_tf, peak_hbm, peak_src = _peaks()
    roof, roof_gemm, roof_ln = _rooflines(log or [], ms_local, peak_tf, peak_hbm, peak_src)
    cpu = None
    if world == 1 and not args.no_cpu_baseline:
        cpu = cpu_baseline(repeats=3, warmup=1)
    xch = "copy-engine peer copies out of symmetric memory" if args.exchange == "peer" else "NCCL all-gather"
    par = (f"temporal-shard x{world} ({T // world} frames/rank), K/V exchanged per layer over NVLink ({xch})" if temporal_main
           else (f"dp{world} (one window per GPU, no collective)" if world > 1 else "single"))
    line = {
        "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": K, "warmup": W,
        "ms_per_step": ms_total / K, "higher_is_better": True, "scaling": scaling, "vs_baseline": None,
        "dtype": "bf16", "data": "synthetic",
        "config": {"workload": WORKLOAD, "parallelism": par, "steps_schedule": "shift 3.0",
                   "l2": "inputs larger than L2 (2.9 GB weights + >3 GB activations per step; no flush needed)",
                   "weights": "seeded random (no checkpoints offline)",
                   "precision": "bf16 GEMM/attention operands, fp32 accumulation, fp32 residual stream"},
        "step_flops": F_STEP, "model_tflops": F_STEP * value / (1 if temporal_main else world) / 1e12,
        "roofline": roof, "roofline_gemm": roof_gemm, "roofline_layernorm": roof_ln,
        "cpu_baseline": cpu,
        "e2e": {"value": e2e_val, "unit": UNIT, "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": d2h,
                "note": "one SchedulerFlow.denoise() call from pinned host buffers incl. per-window context K/V precompute; "
                        "window inputs are copied once (amortised per step), the latents are read back every step"
                        + (" (sharded window: once, after the final all-gather)" if temporal_main else "")},
        "gpu_launches": launches, "clocks": clocks,
    }
    if eager is not None:
        line["gpu_eager_baseline"] = eager
    if other is not None:
        line[other[0]] = other[1]
    if video is not None:
        line["video"] = video
    print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()


NOMINAL_BF16_TF = 989.0    # dense bf16 data-sheet peak of an H100 SXM at 700 W (the roofline denominator prefers a MEASURED figure)
NOMINAL_HBM_GBS = 3350.0   # HBM3 data-sheet bandwidth of an H100 SXM


def _rooflines(log, ms_local, peak_tf, peak_hbm, peak_src):
    """Per-kernel-family roofline entries from the CUDA-event log of the timed region (events on the launching stream)."""
    by = {}
    for tag, e0, e1, meta in log:
        by.setdefault(tag, []).append((e0.elapsed_time(e1), meta))
    attn = by.get("attn_self", [])
    roof = {"bound": "tensor", "kernel": ATTN_KERNEL, "achieved": None, "peak": peak_tf, "unit": "TFLOP/s", "frac": None,
            "traffic": None, "peak_source": peak_src}
    if attn:
        avg_ms = sum(a[0] for a in attn) / len(attn)
        fl = sum(4.0 * m[0] * m[1] * m[2] * m[3] * m[4] for _, m in attn) / len(attn)
        ach = fl / (avg_ms * 1e-3) / 1e12
        roof.update({"achieved": ach, "frac": ach / peak_tf,
                     "launches_timed": len(attn), "avg_launch_ms": avg_ms, "flops_per_launch": fl,
                     "share_of_step": sum(a[0] for a in attn) / ms_local,
                     "frac_of_nominal": ach / NOMINAL_BF16_TF})
    big = [(ms, m) for ms, m in by.get("gemm", []) if m[0] >= 4096]
    rg = None
    if big:
        fl = sum(2.0 * m[0] * m[1] * m[2] for _, m in big)
        tms = sum(ms for ms, _ in big)
        ach = fl / (tms * 1e-3) / 1e12
        rg = {"bound": "tensor", "kernel": "gemm_bf16_kernel (all nn.Linear of the block, fused epilogues)",
              "achieved": ach, "peak": peak_tf, "unit": "TFLOP/s", "frac": ach / peak_tf, "traffic": None,
              "launches_timed": len(big), "share_of_step": tms / ms_local, "frac_of_nominal": ach / NOMINAL_BF16_TF}
    ln = [(ms, m) for ms, m in by.get("layernorm", []) if m[0] >= 4096]
    rl = None
    if ln:
        byts = sum(float(m[0]) * m[1] * m[2] for _, m in ln)
        tms = sum(ms for ms, _ in ln)
        ach = byts / (tms * 1e-3) / 1e9
        rl = {"bound": "hbm", "kernel": "layernorm_kernel", "achieved": ach, "peak": peak_hbm, "unit": "GB/s",
              "frac": ach / peak_hbm, "traffic": None, "launches_timed": len(ln), "share_of_step": tms / ms_local,
              "bytes_per_element": "input + output element sizes (fp32 stream in, bf16 operand out = 6 B)"}
    return roof, rg, rl


def _video_leg(torch, ops, model, cf, dev):
    from actionmesh_b200.scheduler import B200SchedulerFlow

    T, N, C = T_WIN, N_TOK, C_LAT
    video = None
    try:
        import numpy as np
        from PIL import Image

        from actionmesh_b200.image_encoder import B200ImageEncoder
        from actionmesh_b200.pipeline import Stage1Pipeline, VideoInput

        enc = B200ImageEncoder().to(dev)
        enc.init_random_(seed=1235)  # DinoV2-L/14 shape, seeded random weights (no checkpoints offline)
        rng = np.random.default_rng(7)
        frames = [Image.fromarray(rng.integers(0, 255, (512, 512, 3), dtype=np.uint8), "RGB") for _ in range(T)]
        pipe = Stage1Pipeline(model, B200SchedulerFlow(num_inference_steps=30, shift=3.0, is_additive=True), cf, enc)
        anchor = torch.randn(1, N, C, generator=torch.Generator().manual_seed(99))
        vin = VideoInput(frames, torch.arange(T, dtype=torch.float32))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ctx_v = pipe.encode_all_frames(vin)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        bank = pipe(vin, anchor, seed=44, stage_1_steps=30, context=ctx_v)
        lat_out, _ = bank.get_ordered()
        lat_host = lat_out.cpu()
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        video = {"sec_per_video_stage1": t2 - t0, "dinov2_encode_s": t1 - t0, "denoise_30_steps_s": t2 - t1,
                 "frames": T, "steps": 30, "finite": bool(torch.isfinite(lat_host).all()),
                 "note": "Stage-I path only (uint8 frames -> CUDA BitImageProcessor-equivalent preprocessing -> DinoV2 + 1 window x 30 steps, CFG 7.5) through "
                         "Stage1Pipeline; Stage 0 (TripoSG) is out of scope and not included; Stage II is timed separately below"}
        del enc, pipe
        # Stage II (SURVEY 8(f) rank 1) on the same window: 16-block trunk re-run for each of the 15 target times + the
        # fp32-grade vertex-query block for V = 20 000 anchor vertices (+ normals), B200Autoencoder.forward, host in/out.
        from actionmesh_b200.autoencoder import B200Autoencoder

        ae = B200Autoencoder().to(dev)
        ae.init_random_(seed=1236)
        gq = torch.Generator().manual_seed(13)
        pts = torch.randn(1, 20000, 3, generator=gq)
        pts = pts / pts.norm(dim=-1, keepdim=True) * 0.6
        query = torch.cat([pts, pts / 0.6], dim=-1)
        tgt = torch.linspace(0, 1, T)[None, 1:]
        ae.forward(lat_host[None, :3], torch.arange(3.0)[None], torch.zeros(1), tgt[:, :1], query[:, :512])  # warm-up
        ops.event_log, ops.event_tags = [], {"s2_attn", "s2_gemm", "s2_q"}
        torch.cuda.synchronize()
        t3 = time.perf_counter()
        disp = ae.forward(lat_host[None], torch.arange(T, dtype=torch.float32)[None], torch.zeros(1), tgt, query)
        verts = ae.apply_displacement(query[..., :3].to(dev), disp).cpu()
        torch.cuda.synchronize()
        t4 = time.perf_counter()
        s2 = {}
        for tag, e0, e1, _ in ops.event_log:
            s2[tag] = s2.get(tag, 0.0) + e0.elapsed_time(e1)
        ops.event_log = None
        video.update({"stage2_decode_s": t4 - t3, "stage2_targets": int(tgt.shape[1]), "stage2_vertices": 20000,
                      "stage2_kernel_ms": {"trunk_attention": s2.get("s2_attn"), "trunk_gemm": s2.get("s2_gemm"),
                                           "query_path_gemm": s2.get("s2_q")},
                      "stage2_finite": bool(torch.isfinite(verts).all()),
                      "sec_per_video_stage1_plus_stage2": (t2 - t0) + (t4 - t3)})
        del ae
    except Exception as exc:  # noqa: BLE001 - an optional leg must never cost the main JSON line
        ops.event_log = None
        video = dict(video or {}, error=f"{type(exc).__name__}: {exc}"[:400])
    return video


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--mode", default="temporal", choices=["temporal", "dp"])
    ap.add_argument("--exchange", default="peer", choices=["nccl", "peer"],
                    help="per-layer K/V exchange of the sharded window: NCCL all-gather or copy-engine peer copies")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-video", action="store_true")
    ap.add_argument("--no-eager", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the denoised latents of the timed window to DIR/latents.npy (float32)")
    args = ap.parse_args()
    if args.impl == "reference":
        run_reference(args, int(os.environ.get("RANK", "0")))
        return
    run_b200(args)


if __name__ == "__main__":
    main()
