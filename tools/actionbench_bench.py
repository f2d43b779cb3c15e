"""Time ActionBench's gradient ICP and a whole CD-3D / CD-4D / CD-M clip on the GPU; print one JSON line.

    python tools/actionbench_bench.py [--runs 3] [--eager-runs 1] [--out results/actionbench_bench.json]

  * the card's name and power limit, read in the same run;
  * per-iteration kernel time of one ICP step (icp_chamfer_grad + icp_adam_step) at F = 16 frames, C = 24 candidates,
    P = Q = 10 000 points, from CUDA events over 50 steps after 10 warm-up steps, and point pairs per second
    (2 F C P Q per step);
  * seconds per clip: compute_chamfer_3d_4d(is_4D=True) on 16 frames of a synthetic deforming mesh of ~20 000 faces with
    the benchmark's sizes (10 000 ICP points, 100 000 Chamfer points), one warm-up clip, then the median of --runs;
  * the same clip's ICP through a torch-eager restatement of the reference's loop (`eager_gradient_icp`: cdist Chamfer,
    autograd, torch.optim.Adam and a `.item()` per step, 17 runs as benchmark.py makes them) on the same GPU.  This is a
    restatement of the reference's algorithm in eager PyTorch, not pytorch3d.
The lower bound from counts is 16 runs x 200 steps x 2 x 24 x 10^8 pairs = 1.5e13 pairs per clip.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _rot6d(d6: torch.Tensor) -> torch.Tensor:
    a1, a2 = d6[..., :3], d6[..., 3:]
    b1 = torch.nn.functional.normalize(a1, dim=-1)
    b2 = torch.nn.functional.normalize(a2 - (b1 * a2).sum(-1, keepdim=True) * b1, dim=-1)
    return torch.stack((b1, b2, torch.cross(b1, b2, dim=-1)), dim=-2)


@torch.enable_grad()
def eager_gradient_icp(pc_pred, pc_gt, lr: float = 0.01, n_iter: int = 200, with_history: bool = False):
    """icp.py:53-112 restated in eager torch (cdist-based Chamfer, autograd, torch.optim.Adam, a host sync per step) ->
    best (16,) = loss, R, T, s as the reference records them (R before the step, T and s after it)."""
    from actionmesh_b200.evaluation import canonical_rotation_matrices

    dev = pc_pred.device
    R_init = canonical_rotation_matrices().to(dev)
    n = len(R_init)
    pred, gt = pc_pred[None].expand(n, -1, -1), pc_gt[None].expand(n, -1, -1)
    T = torch.nn.Parameter(torch.zeros(n, 3, device=dev))
    d6 = torch.nn.Parameter(torch.tensor([[1.0, 0.0, 0.0, 0.0, 1.0, 0.0]], device=dev).repeat(n, 1))
    s = torch.nn.Parameter(torch.ones(n, 3, device=dev))
    opt = torch.optim.Adam(params=[T, d6, s], lr=lr)
    best_loss, best, history = float("inf"), None, []
    for _ in range(n_iter):
        opt.zero_grad()
        R = R_init @ _rot6d(d6)
        y = s[:, None] * pred @ R + T[:, None]
        d = torch.cdist(y, gt) ** 2
        loss = d.min(2).values.mean(1) + d.min(1).values.mean(1)
        loss.mean().backward()
        opt.step()
        min_loss, idx = loss.detach().min(0)
        if min_loss.item() < best_loss:
            best_loss = min_loss.item()
            best = torch.cat([min_loss[None], R[idx].detach().reshape(9), T[idx].detach(), s[idx].detach()])
        history.append(best_loss)
    return (best, torch.tensor(history)) if with_history else best


def synthetic_clip(frames: int = 16, lat: int = 100, lon: int = 100):
    """A latitude-longitude ellipsoid (2 lon (lat - 1) = 19 800 faces) bending over the frames, and ground truth sampled
    from the same animation under a similarity transform."""
    verts = [[0.0, 0.0, 1.0]]
    th = np.pi * np.arange(1, lat) / lat
    ph = 2 * np.pi * np.arange(lon) / lon
    ring = np.stack([np.outer(np.sin(th), np.cos(ph)), np.outer(np.sin(th), np.sin(ph)),
                     np.outer(np.cos(th), np.ones(lon))], -1).reshape(-1, 3)
    verts = np.concatenate([verts, ring, [[0.0, 0.0, -1.0]]]) * np.array([1.0, 0.6, 0.4])
    idx = lambda i, j: 1 + (i - 1) * lon + j % lon  # noqa: E731
    faces = []
    for j in range(lon):
        faces += [[0, idx(1, j), idx(1, j + 1)], [len(verts) - 1, idx(lat - 1, j + 1), idx(lat - 1, j)]]
    for i in range(1, lat - 1):
        for j in range(lon):
            faces += [[idx(i, j), idx(i + 1, j), idx(i + 1, j + 1)], [idx(i, j), idx(i + 1, j + 1), idx(i, j + 1)]]
    faces = np.array(faces, dtype=np.int64)
    meshes = []
    for t in range(frames):
        v = verts.copy()
        v[:, 2] += 0.02 * t * v[:, 0] ** 2
        v[:, 1] += 0.01 * t
        meshes.append(SimpleNamespace(vertices=v, faces=faces))
    from actionmesh_b200.evaluation import sample_meshes

    gt = sample_meshes(meshes, n_pts=100_000, synchronized=True, seed=5)
    c, s_ = np.cos(0.3), np.sin(0.3)
    R = torch.tensor([[c, -s_, 0.0], [s_, c, 0.0], [0.0, 0.0, 1.0]], dtype=torch.float32)
    gt = (gt * torch.tensor([1.1, 0.95, 1.05])) @ R + torch.tensor([0.05, -0.02, 0.03])
    return meshes, gt


def _card() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (x.strip() for x in q.split(","))
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as exc:  # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(), "power_limit": f"unknown ({exc})"}


def kernel_step_time(F=16, C=24, P=10_000, Q=10_000, warmup=10, steps=50) -> dict:
    from actionmesh_b200 import ops
    from actionmesh_b200.evaluation import canonical_rotation_matrices

    gen = torch.Generator().manual_seed(0)
    x = (torch.randn(F, P, 3, generator=gen) * torch.tensor([1.0, 0.6, 0.4])).cuda()
    g = (torch.randn(F, Q, 3, generator=gen) * torch.tensor([1.0, 0.6, 0.4])).cuda()
    rot_init = canonical_rotation_matrices().cuda()
    params = torch.zeros(F, C, 12, device="cuda")
    params[..., 3] = params[..., 7] = 1.0
    params[..., 9:] = 1.0
    rot = rot_init.repeat(F, 1, 1, 1)
    m, v = torch.zeros_like(params), torch.zeros_like(params)
    best = torch.full((F, 16), float("inf"), device="cuda")
    sums = torch.empty(F, C, 13, dtype=torch.float64, device="cuda")
    scratch = torch.empty(ops.icp_scratch_doubles(F, C, P, Q), dtype=torch.float64, device="cuda")

    def step(i):
        ops.icp_chamfer_grad(x, g, rot, params, out=sums, scratch=scratch)
        ops.icp_adam_step(sums, rot_init, i + 1, 0.01, params, m, v, rot, best)

    for i in range(warmup):
        step(i)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        step(warmup + i)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    pairs = 2 * F * C * P * Q
    return {"F": F, "C": C, "P": P, "Q": Q, "ms_per_step": ms, "pairs_per_step": pairs,
            "pairs_per_s": pairs / (ms * 1e-3)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--eager-runs", type=int, default=1)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("actionbench_bench: no CUDA device (this measures the GPU; there is nothing to time on the CPU)")
    from actionmesh_b200.evaluation import compute_chamfer_3d_4d, sample_meshes, sample_point_cloud

    res = _card()
    res["kernel"] = kernel_step_time()

    meshes, gt = synthetic_clip()
    scores, times = None, []
    for r in range(a.runs + 1):                   # run 0 warms up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        scores = compute_chamfer_3d_4d(gt, meshes, device="cuda", is_4D=True)
        torch.cuda.synchronize()
        if r:
            times.append(time.perf_counter() - t0)
    res["clip"] = {"frames": len(meshes), "faces": int(len(meshes[0].faces)), "seconds": statistics.median(times),
                   "all_seconds": times, "scores": scores}

    # the reference's 17 ICP runs (16 per-frame + 1 unified) through the eager restatement, on the same inputs
    pred_icp = sample_point_cloud(sample_meshes(meshes, n_pts=100_000, synchronized=False, seed=44), 10_000, 44).cuda()
    gt_icp = sample_point_cloud(gt, 10_000, 44).cuda()
    eager = []
    for _ in range(a.eager_runs):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for k in list(range(len(meshes))) + [0]:
            eager_gradient_icp(pred_icp[k], gt_icp[k])
        torch.cuda.synchronize()
        eager.append(time.perf_counter() - t0)
    res["eager_icp_restatement"] = {"what": "torch-eager restatement of the reference's gradient_icp loop (cdist Chamfer, "
                                            "autograd, Adam, .item() per step), 17 runs; not pytorch3d",
                                    "seconds": statistics.median(eager), "all_seconds": eager}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
