"""Run BASELINE.json's configurations c3 / c4 / c5 at their named shapes (seeded random weights, synthetic frames) and print
one JSON line each; c1 (8 frames, 4 steps, full width) is the parity test tests/test_default_config_gpu.py, c2 is bench.py.

    python tools/run_config.py c3                                   # 1 GPU: --fast (15 steps), 32 frames = 3 AR windows
    torchrun --nproc-per-node 8 tools/run_config.py c4 --clips 16   # whole-clip data parallel (the config names 128 clips)
    torchrun --nproc-per-node 8 tools/run_config.py c5              # 256 frames = 17 serial windows, each frame-sharded 8-way

Timed with CUDA events around the Stage-I loop (DinoV2 context included for c3), max over ranks."""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    import torch.distributed as dist

    ap = argparse.ArgumentParser()
    ap.add_argument("config", choices=["c3", "c4", "c5"])
    ap.add_argument("--clips", type=int, default=16)
    ap.add_argument("--steps", type=int, default=None)
    ap.add_argument("--exchange", default="peer", choices=["nccl", "peer"])
    args = ap.parse_args()
    rank, local, world = (int(os.environ.get(k, d)) for k, d in (("RANK", 0), ("LOCAL_RANK", 0), ("WORLD_SIZE", 1)))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    from actionmesh_b200.denoiser import B200Denoiser, DenoiserConfig
    from actionmesh_b200.guidance import ClassifierFreeGuidance
    from actionmesh_b200.pipeline import Stage1Pipeline, VideoInput
    from actionmesh_b200.scheduler import B200SchedulerFlow
    from actionmesh_b200.windows import LatentBank, chunk_from

    shard = None
    if world > 1:
        from actionmesh_b200.window_shard import FrameShard, PeerFrameShard, configure_nccl_env

        configure_nccl_env()
        dist.init_process_group("nccl", device_id=dev)
        if args.config == "c5":
            shard = PeerFrameShard() if args.exchange == "peer" else FrameShard()
    model = B200Denoiser(DenoiserConfig()).to(dev)
    model.init_random_(seed=1234)
    cf = ClassifierFreeGuidance(guidance_at_inference=[[0, 1], [1, 1]], guidance_scales=[7.5])
    N, C, S, Dc = 2048, 64, 257, 1024

    def sync():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def run_clip(n_frames, steps, seed, context, use_shard):
        """Stage I of one clip through the AR windows of generate_3d_latents (pipeline.py:435-508)."""
        sch = B200SchedulerFlow(num_inference_steps=steps, shift=3.0, is_additive=True)
        pipe = Stage1Pipeline(model, sch, cf, image_encoder=None)
        ts = torch.arange(n_frames, dtype=torch.float32)
        bank = LatentBank(empty_dims=(N, C))
        anchor = torch.randn(1, N, C, generator=torch.Generator().manual_seed(99 + seed))
        bank.update(timesteps=ts[0:1], latents=anchor.to(dev))
        vin = VideoInput([None] * n_frames, ts)
        if not use_shard:
            return pipe.generate_3d_latents(vin, context, bank, seed=seed)
        windows = chunk_from(start=0, total=n_frames, size=16, slide=15)
        for i, idx in enumerate(windows):   # Stage1Pipeline._denoise_latents with the window frame-sharded over the ranks
            win = vin.get(idx)
            gen = torch.Generator(device=dev).manual_seed(seed + i)
            cond, cmask = bank.get(timesteps=win.timesteps, device=dev, add_batch_dim=True)
            noise = sch.get_noise(batch_size=1, latent_shape=[N, C], n_timesteps=win.n_frames, generator=gen, device=dev)
            m = cmask[..., None, None].to(torch.float32)
            lat = sch.denoise(model, cf, cond * m + noise * (1.0 - m), context[idx.to(dev)][None], mask=cmask.to(torch.float32),
                              framestep=win.timesteps[None], device=dev, shard=shard)
            bank.update(latents=lat, timesteps=win.timesteps)
        return bank

    if args.config == "c3":
        n_frames, steps = 32, args.steps or 15
        ctx = torch.randn(n_frames, S, Dc, generator=torch.Generator().manual_seed(5)).to(dev)
        n_windows = len(chunk_from(0, n_frames, 16, 15))
        run_clip(16, 1, 0, ctx[:16], False)                       # warm-up (workspace allocation, kernel attributes)
        sync()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        bank = run_clip(n_frames, steps, 44, ctx, False)
        e1.record()
        sync()
        lat, _ = bank.get_ordered()
        out = {"config": "c3: --fast scheduler (15 steps), 32-frame synthetic video, bf16 operands, 1xH100", "frames": n_frames,
               "windows": n_windows, "steps_per_window": steps, "denoiser_steps": n_windows * steps,
               "stage1_seconds": e0.elapsed_time(e1) / 1e3, "steps_per_sec": n_windows * steps / (e0.elapsed_time(e1) / 1e3),
               "finite": bool(torch.isfinite(lat).all()), "latents_shape": list(lat.shape),
               "note": "windows 2 and 3 hold 1 and 15 observed frames (chunk_from(0,32,16,15)): same work per step as a full window"}
    elif args.config == "c4":
        steps = args.steps or 30
        per_rank = max(1, args.clips // world)
        ctx = torch.randn(16, S, Dc, generator=torch.Generator().manual_seed(5 + rank)).to(dev)
        run_clip(16, 1, 0, ctx, False)
        sync()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for c in range(per_rank):
            run_clip(16, steps, 1000 * rank + c, ctx, False)
        e1.record()
        sync()
        t = torch.tensor([e0.elapsed_time(e1)], device=dev, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        sec = float(t.item()) / 1e3
        out = {"config": f"c4: ActionBench-style batch, whole-clip data parallel across {world}xH100 (no data-path collective)",
               "clips_run": per_rank * world, "clips_per_gpu": per_rank, "steps_per_clip": steps, "seconds": sec,
               "clips_per_sec": per_rank * world / sec, "denoiser_steps_per_sec": per_rank * world * steps / sec,
               "projected_seconds_128_clips": 128 / (per_rank * world / sec)}
    else:
        n_frames, steps = 256, args.steps or 30
        ctx = torch.randn(n_frames, S, Dc, generator=torch.Generator().manual_seed(5)).to(dev)
        windows = chunk_from(0, n_frames, 16, 15)
        run_clip(16, 1, 0, ctx[:16], shard is not None)
        sync()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        bank = run_clip(n_frames, steps, 44, ctx, shard is not None)
        e1.record()
        sync()
        t = torch.tensor([e0.elapsed_time(e1)], device=dev, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        sec = float(t.item()) / 1e3
        lat, _ = bank.get_ordered()
        out = {"config": f"c5: single 256-frame synthetic video, 17 serial AR windows, each window's frames sharded across {world}xH100 "
                         f"({'copy-engine peer copies' if args.exchange == 'peer' else 'NCCL all-gather'} of the temporal-attention K/V)",
               "frames": n_frames, "windows": len(windows), "steps_per_window": steps, "denoiser_steps": len(windows) * steps,
               "seconds": sec, "steps_per_sec": len(windows) * steps / sec, "finite": bool(torch.isfinite(lat).all()),
               "frames_denoised": int(lat.shape[0])}
    if rank == 0:
        print(json.dumps(out), flush=True)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
