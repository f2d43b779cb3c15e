"""Frame-sharded window (-m gpu): the sharded denoise over W ranks with the per-layer K/V all-gather must equal the
single-GPU denoise of the same window (same kernels, different chunking of the key loop => only accumulation-order noise:
rel <= 5e-3), observed frames bit-identical.

* `test_sharded_program_emulated_on_one_gpu`: W = 2, 4, 8 ranks EMULATED on one GPU — one host thread per rank runs the
  unmodified `B200SchedulerFlow.denoise(..., shard=...)` with a `LocalShard` whose gathers are device copies between the
  ranks' buffers (threading barriers stand in for the collective's rendezvous).  Covers frame slicing, the staggered
  per-branch programs, the `kv_chunks` attention path and the latent gather end to end on the driver's 1-GPU box.
* `test_sharded_window_matches_single_gpu`: the real thing over NCCL (needs >= 2 devices)."""
import os
import socket
import threading

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    from actionmesh_b200.window_shard import configure_nccl_env

    configure_nccl_env()
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from actionmesh_b200.denoiser import B200Denoiser, DenoiserConfig
        from actionmesh_b200.guidance import ClassifierFreeGuidance
        from actionmesh_b200.scheduler import B200SchedulerFlow
        from actionmesh_b200.window_shard import FrameShard, PeerFrameShard
        from oracle import synth

        d = dict(num_layers=3, num_attention_heads=2, width=256, cross_attention_dim=128, in_channels=64, mlp_ratio=4.0)
        cfg = DenoiserConfig(inflated_layers=(0, 2), **d)  # one non-inflated layer exercises the local path too
        model = B200Denoiser(cfg).to(f"cuda:{rank}")
        model.load_state_dict(synth.make_state_dict(cfg, 3))
        lat, ctx, fs, mask = synth.make_inputs(1, 4, 63, 64, 9, 128, seed=8)
        sch = B200SchedulerFlow(num_inference_steps=3, shift=3.0, is_additive=True)
        cf = ClassifierFreeGuidance(guidance_at_inference=[[0, 1], [1, 1]], guidance_scales=[7.5])
        dev = f"cuda:{rank}"
        ref = sch.denoise(model, cf, lat.clone().to(dev), ctx.to(dev), mask=mask.to(dev), framestep=fs)
        res = []
        for kind in (FrameShard, PeerFrameShard):   # NCCL all-gather / copy-engine peer copies out of symmetric memory
            out = sch.denoise(model, cf, lat.clone().to(dev), ctx.to(dev), mask=mask.to(dev), framestep=fs, shard=kind())
            err = float((out - ref).norm() / ref.norm())
            res.append(err < 5e-3 and torch.equal(out[0, 0].cpu(), lat[0, 0]))
            if not res[-1]:
                res[-1] = f"{kind.__name__} err {err}"
        q.put((rank, "ok" if all(r is True for r in res) else str(res)))
    except Exception:  # noqa: BLE001
        import traceback

        q.put((rank, traceback.format_exc()[-1500:]))
    finally:
        dist.destroy_process_group()


class _LocalWorld:
    def __init__(self, world):
        self.world = world
        self.barrier = threading.Barrier(world)
        self.slots = [None] * world


class LocalShard:
    """Stand-in for window_shard.FrameShard with every rank living in one process on one GPU (test infrastructure)."""

    def __init__(self, lw: _LocalWorld, rank: int):
        self.lw, self.rank, self.world, self.slot, self.group = lw, rank, lw.world, rank, None

    def frames(self, n_frames):
        from actionmesh_b200.window_shard import frame_partition

        return frame_partition(n_frames, self.world, self.rank)

    def _exchange(self, local):
        lw = self.lw
        lw.slots[self.rank] = local
        lw.barrier.wait()                      # every rank has launched the kernels producing its `local`
        parts = list(lw.slots)
        return parts

    def all_gather_kv(self, out, local, channel=0):
        parts = self._exchange(local)
        rows = local.shape[0]
        for r, part in enumerate(parts):       # same stream as the producers: ordered after them
            out[r * rows:(r + 1) * rows].copy_(part)
        self.lw.barrier.wait()                 # nobody overwrites its `local` before every copy has been enqueued

        class _Done:
            def wait(self_inner):
                return None

        return _Done()

    def gather_latents(self, local):
        parts = self._exchange(local)
        out = torch.cat(list(parts), dim=1).clone()
        self.lw.barrier.wait()
        return out


@pytest.mark.parametrize("world", [2, 4, 8])
def test_sharded_program_emulated_on_one_gpu(amb_lib, world):
    from actionmesh_b200.denoiser import B200Denoiser, DenoiserConfig
    from actionmesh_b200.guidance import ClassifierFreeGuidance
    from actionmesh_b200.scheduler import B200SchedulerFlow
    from oracle import synth

    d = dict(num_layers=3, num_attention_heads=2, width=256, cross_attention_dim=128, in_channels=64, mlp_ratio=4.0)
    cfg = DenoiserConfig(inflated_layers=(0, 2), **d)  # one non-inflated layer exercises the local path too
    model = B200Denoiser(cfg).to("cuda")
    model.load_state_dict(synth.make_state_dict(cfg, 3))
    lat, ctx, fs, mask = synth.make_inputs(1, 8, 63, 64, 9, 128, seed=8)
    sch = B200SchedulerFlow(num_inference_steps=3, shift=3.0, is_additive=True)
    cf = ClassifierFreeGuidance(guidance_at_inference=[[0, 1], [1, 1]], guidance_scales=[7.5])
    ref = sch.denoise(model, cf, lat.clone().cuda(), ctx.cuda(), mask=mask.cuda(), framestep=fs).cpu()
    lw = _LocalWorld(world)
    outs, errs = [None] * world, []

    def run(rank):
        try:
            torch.cuda.set_device(0)
            outs[rank] = sch.denoise(model, cf, lat.clone().cuda(), ctx.cuda(), mask=mask.cuda(), framestep=fs,
                                     shard=LocalShard(lw, rank)).cpu()
        except Exception as exc:  # noqa: BLE001
            errs.append((rank, repr(exc)[:400]))
            lw.barrier.abort()

    threads = [threading.Thread(target=run, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=300)
    assert not errs, errs
    errors = [float((outs[r] - ref).norm() / ref.norm()) for r in range(world)]
    # When a rank's chunk is a whole number of 128-key tiles the sharded key loop visits the same tiles in the same order
    # as the single-GPU loop: bit-identical.  With 1 frame (64 keys) per rank every tile is a ragged half tile, a different
    # but equally valid summation order; three CFG-7.5 steps amplify that like any other rounding difference, so the bar
    # there is the distance to the fp32 oracle: the sharded result may not be further from it than the single-GPU result.
    from oracle import denoiser_oracle as do

    ocfg = do.DenoiserConfig(inflated_layers=(0, 2), **d)
    truth = do.flow_denoise(do.OracleDenoiser(synth.make_state_dict(cfg, 3), ocfg), lat, ctx, mask, fs,
                            num_inference_steps=3, guidance_scales=[7.5])
    e_single = float((ref - truth).norm() / truth.norm())
    e_shard = float((outs[0] - truth).norm() / truth.norm())
    print("SHARD_EMULATION", world, errors[0], "vs oracle: single", e_single, "sharded", e_shard)
    aligned = (lat.shape[1] // world) * (lat.shape[2] + 1) % 128 == 0
    for r in range(world):
        assert errors[r] < (5e-3 if aligned else 3e-2), (r, errors)
        assert torch.equal(outs[r][0, 0], lat[0, 0])   # the observed frame comes back bit-identical on every rank
    assert e_shard <= 1.25 * e_single + 1e-3, (e_single, e_shard)
    assert all(torch.equal(outs[0], o) for o in outs[1:])  # every rank ends with the same full window


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_sharded_window_matches_single_gpu(amb_lib):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, "ok"), (1, "ok")], res
