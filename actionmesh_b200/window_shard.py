"""Temporal (frame) sharding of ONE 16-frame denoising window across the GPUs of a box (SURVEY 8(e), config 5).

Everything in a DiT block is token-local — LayerNorm, QKV / out / MLP GEMMs, the cross-attention to the frame's own 257
context tokens (temporal_denoiser.py:221-226), the skip linears, the time token — except the inflated self-attention,
where every query attends to the keys of all T·L tokens (attention_processor.py:49-65).  So each rank owns T/world
consecutive frames of every CFG branch, keeps its queries local, and per layer all-gathers K and V (post RMSNorm/RoPE,
bf16) over NCCL.  The attention kernel consumes the gathered buffer in place as `kv_chunks = world` chunks (5-D TMA map
with a free chunk stride; no re-layout).  The fp32 latents are sharded the same way and all-gathered once per window.

One process per GPU (`torch.distributed`, backend "nccl" on the box, "gloo" in the CPU tests of the index logic).
"""
from __future__ import annotations

import os
from typing import Optional

import torch
import torch.distributed as dist


def frame_partition(n_frames: int, world: int, rank: int) -> slice:
    """Frames [rank*T/world, (rank+1)*T/world).  T must divide evenly (16 frames over 1/2/4/8 ranks)."""
    if n_frames % world:
        raise ValueError(f"{n_frames} frames do not shard evenly over {world} ranks")
    per = n_frames // world
    return slice(rank * per, (rank + 1) * per)


def gather_kv(kv_local: torch.Tensor, group=None) -> torch.Tensor:
    """All-gather the local (B*T_local*L, 2D) [K|V] rows of one layer -> (world, B*T_local*L, 2D), rank-major."""
    world = dist.get_world_size(group)
    out = torch.empty((world,) + tuple(kv_local.shape), dtype=kv_local.dtype, device=kv_local.device)
    dist.all_gather_into_tensor(out.view(-1, kv_local.shape[-1]), kv_local.contiguous(), group=group)  # concat along dim 0
    return out


def chunked_kv_views(kv_all: torch.Tensor, B: int, s_local: int, H: int, dh: int):
    """(world, B*s_local, 2*H*dh) gathered buffer -> K, V views of logical shape (B, world, s_local, H, dh): chunk c of
    batch b is rank c's keys; concatenating the chunks in rank order restores the window's frame order."""
    world = kv_all.shape[0]
    D = H * dh
    kv5 = kv_all.view(world, B, s_local, 2 * D).permute(1, 0, 2, 3)  # (B, world, s_local, 2D), no copy
    k = kv5[..., 0:D].unflatten(-1, (H, dh))
    v = kv5[..., D:2 * D].unflatten(-1, (H, dh))
    return k, v


def configure_nccl_env() -> None:
    """Defaults for the per-layer K/V all-gather; call BEFORE `init_process_group` (NCCL caches its parameters at first use).
    The Simple protocol on 32 channels was chosen on the project's first (Blackwell) target, where it cut the exposed gather
    time per step about tenfold against NCCL's default choice (tools/shard_profile.py shows the timeline); it has not been
    re-measured on H100s.  Explicit user settings win (setdefault)."""
    os.environ.setdefault("NCCL_PROTO", "Simple")
    os.environ.setdefault("NCCL_MIN_NCHANNELS", "32")


class _EventWork:
    """`.wait()` with the semantics of an async NCCL work handle: the CURRENT stream waits for the recorded event."""

    def __init__(self, event):
        self.event = event

    def wait(self):
        torch.cuda.current_stream().wait_event(self.event)


class FrameShard:
    """Rank-local view of a frame-sharded window, handed to B200Denoiser._forward_packed.  The per-layer K/V exchange is an
    NCCL all-gather on a dedicated high-priority communicator; `PeerFrameShard` replaces it with copy-engine peer copies."""

    def __init__(self, group=None):
        if group is None and dist.get_backend() == "nccl":
            # dedicated communicator on a HIGH-PRIORITY stream: the per-layer K/V all-gather has to run concurrently with
            # compute kernels that fill every SM (persistent GEMMs, multi-wave attention); at normal priority its CTAs
            # queue behind the pending compute CTAs and the gather is effectively serialised.
            opts = dist.ProcessGroupNCCL.Options(is_high_priority_stream=True)
            group = dist.new_group(ranks=list(range(dist.get_world_size())), pg_options=opts)
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)

    def frames(self, n_frames: int) -> slice:
        return frame_partition(n_frames, self.world, self.rank)

    def all_gather_kv(self, out: torch.Tensor, local: torch.Tensor, channel: int = 0):
        """Asynchronous all-gather of this rank's (rows, 2D) [K|V] of one layer/branch into `out` (world*rows, 2D),
        rank-major; returns a handle whose `.wait()` makes the current stream wait for it.  `channel` = the CFG branch."""
        return dist.all_gather_into_tensor(out, local, group=self.group, async_op=True)

    def gather_latents(self, local: torch.Tensor) -> torch.Tensor:
        """(1, T_local, N, C) fp32 per rank -> (1, T, N, C) on every rank (once per window)."""
        out = torch.empty((self.world,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
        dist.all_gather_into_tensor(out.view(-1, *local.shape[2:]), local[0].contiguous(), group=self.group)
        return out.reshape(1, -1, *local.shape[2:])


class PeerFrameShard(FrameShard):
    """The per-layer K/V exchange over NVLink peer memory with the COPY ENGINES instead of an NCCL kernel.

    Why: next to SM-filling compute (persistent GEMMs, multi-wave attention) the cost of the all-gather is not its latency
    but its SMs — NCCL's 32-channel kernel runs concurrently with the other CFG branch's attention / MLP and inflates their
    time (timeline: tools/shard_profile.py).  DMA copies take no SM.

    How: every rank's K/V projection writes into a symmetric-memory buffer (torch.distributed._symmetric_memory: one
    allocation per rank, mapped into every peer; `empty_kv_local` hands it to the denoiser's workspace).  `all_gather_kv`
    then, on a side stream: wait for the projection -> device-side barrier across ranks (every rank's projection of this
    layer / branch is complete) -> `world` contiguous peer->local copies (cudaMemcpyAsync D2D, own chunk first, peers in a
    rank-rotated order so each NVLink port sees one reader at a time) -> event the attention launch waits on.
    The local buffer is double-buffered by use parity: a rank writes parity p again two exchanges of the same branch later,
    after it passed the barrier of the exchange in between, which every peer enters only after its own copies of this one
    (stream order on its side stream)."""

    def __init__(self, group=None):
        super().__init__(group)
        self._bufs = {}
        self._uses = {}
        self.stream = None

    @staticmethod
    def available(device) -> bool:
        """Collective probe: can every rank allocate symmetric memory on its device?  (All ranks get the same answer, so a
        caller may choose the NCCL exchange instead without the ranks diverging.)"""
        ok = 1
        try:
            import torch.distributed._symmetric_memory as symm_mem

            symm_mem.empty((1024,), dtype=torch.bfloat16, device=device)
        except Exception:  # noqa: BLE001 - any allocator / driver refusal means "not available"
            ok = 0
        flag = torch.tensor([ok], dtype=torch.int32, device=device)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        return bool(flag.item())

    def empty_kv_local(self, rows: int, cols: int, device) -> torch.Tensor:
        """(2, rows, cols) bf16 symmetric buffer; index [parity] is what the K/V projection of an exchange writes."""
        import torch.distributed._symmetric_memory as symm_mem

        key = (rows, cols)
        if key not in self._bufs:
            group = self.group if self.group is not None else dist.group.WORLD
            buf = symm_mem.empty((2, rows, cols), dtype=torch.bfloat16, device=device)
            hdl = symm_mem.rendezvous(buf, group)
            peers = [buf if r == self.rank else hdl.get_buffer(r, (2, rows, cols), torch.bfloat16) for r in range(self.world)]
            self._bufs[key] = (buf, hdl, peers)
            self.stream = torch.cuda.Stream(device=device, priority=-1)
        return self._bufs[key][0]

    def kv_local_view(self, buf: torch.Tensor, rows: slice, channel: int) -> torch.Tensor:
        """The rows of `buf` the next exchange on `channel` (= CFG branch) will send (alternating parity)."""
        return buf[self._uses.get(channel, 0) & 1, rows]

    def all_gather_kv(self, out: torch.Tensor, local: torch.Tensor, channel: int = 0):
        key = next(k for k, v in self._bufs.items() if v[0].data_ptr() <= local.data_ptr() < v[0].data_ptr() + v[0].numel() * 2)
        buf, hdl, peers = self._bufs[key]
        off = (local.data_ptr() - buf.data_ptr()) // 2
        n = local.numel()
        rows = local.shape[0]
        ready = torch.cuda.Event()
        ready.record(torch.cuda.current_stream())
        self._uses[channel] = self._uses.get(channel, 0) + 1
        with torch.cuda.stream(self.stream):
            self.stream.wait_event(ready)
            hdl.barrier(channel=channel)
            for k in range(self.world):
                r = (self.rank + k) % self.world
                src = peers[r].view(-1)[off:off + n].view(rows, -1)
                out[r * rows:(r + 1) * rows].copy_(src, non_blocking=True)
            done = torch.cuda.Event()
            done.record(self.stream)
        return _EventWork(done)
