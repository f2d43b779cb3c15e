"""One-GPU simulation of ONE rank of a `world`-way frame-sharded window (development tool, not part of the product):
the NCCL all-gather is replaced by a no-op (K/V chunks of the other ranks are random), so the time measured is the
rank's pure compute + launch cost.  Compared with the real multi-GPU `temporal_shard` bench line it tells how much of
the step is communication exposure.  Also prints the host-side issue time of one step (launch-bound check)."""
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from actionmesh_b200 import ops  # noqa: E402
from actionmesh_b200.denoiser import B200Denoiser  # noqa: E402


class _Done:
    def wait(self):
        return True


class FakeShard:
    def __init__(self, world):
        self.world, self.rank, self.group = world, 0, None

    def all_gather_kv(self, out, local, channel=0):
        return _Done()


def main():
    world = int(sys.argv[1]) if len(sys.argv) > 1 else 8
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 4
    dev = torch.device("cuda:0")
    model = B200Denoiser().to(dev)
    model.init_random_(1234)
    T_all, N, C = 16, 2048, 64
    T = T_all // world
    B = 2
    g = torch.Generator().manual_seed(5)
    ctx = torch.randn(1, T_all, 257, 1024, generator=g)
    ctx = torch.cat([torch.zeros_like(ctx), ctx]).to(dev)
    fs = torch.arange(T_all, dtype=torch.float32)[None].repeat(B, 1)
    st = model.precompute_window(ctx, fs, N, frame_slice=slice(0, T))
    ws = model._workspace(B, T, N, world=world)
    ws["kv_all"].normal_()
    ws["x_in"].normal_()
    t32 = torch.full((1,), 500.0, device=dev)
    m32 = torch.zeros(B * T, device=dev)
    shard = FakeShard(world)
    for rep in range(2):
        for _ in range(2):
            model._forward_packed(ws, st, B, T, N, t32, m32, n_input_branches=1, shard=shard)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        l0 = ops.launch_count
        e0.record()
        h0 = time.perf_counter()
        for _ in range(steps):
            model._forward_packed(ws, st, B, T, N, t32, m32, n_input_branches=1, shard=shard)
        h1 = time.perf_counter()
        e1.record()
        torch.cuda.synchronize()
        print(f"world={world} run {rep}: {e0.elapsed_time(e1) / steps:.2f} ms/step on the device, "
              f"host issue {1e3 * (h1 - h0) / steps:.2f} ms/step, {(ops.launch_count - l0) // steps} launches/step", flush=True)


if __name__ == "__main__":
    main()
