"""Regenerate tests/golden/actionbench_tiny.pt from the reference's OWN ActionBench code.

    ACTIONMESH_REFERENCE=/path/to/actionmesh python tools/gen_actionbench_golden.py

Needs a checkout of facebookresearch/actionmesh: actionbench/{icp,sample_mesh,sample_point_cloud,benchmark,chamfer}.py are
imported unchanged on top of oracle/pytorch3d_shim.py.  trimesh is stubbed: `Trimesh` holds vertices and faces, and
`sample.sample_surface` is mesh_input.sample_surface_points (the restatement of trimesh's sampler).  Stored:
  * gradient_icp on two asymmetric clouds of 256 and 240 points: R, T, s of the result and the best loss after every step;
  * canonical_rotation_matrices();
  * sample_meshes in both modes on a small deforming mesh (4 frames), with the synchronized face indices, and a
    sample_point_cloud subsample;
  * compute_chamfer_3d_4d(is_4D=True) on those 4 frames with n_pts_icp = 256, n_pts_chamfer = 2000.
The reference's gradient_icp takes a few seconds per run on the CPU at these sizes.  `--rerun-icp OUT` re-runs the stored
gradient_icp case and writes its result to OUT (tests/test_actionbench_cpu.py checks it against the golden).
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import pytorch3d_shim, reference_loader  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "actionbench_tiny.pt")
SEED = 44
N_ITER = 200


class _Trimesh:
    def __init__(self, vertices, faces):
        self.vertices, self.faces = np.asarray(vertices, dtype=np.float64), np.asarray(faces, dtype=np.int64)


def _install_stubs():
    from actionmesh_b200.mesh_input import sample_surface_points

    pytorch3d_shim.install()
    tm = types.ModuleType("trimesh")
    tm.Trimesh = _Trimesh
    tm.sample = types.SimpleNamespace(
        sample_surface=lambda mesh, count, seed=None: sample_surface_points(mesh.vertices, mesh.faces, count, seed))
    tm._AMB_SHIM = True
    sys.modules["trimesh"] = tm
    # sample_mesh.py forks the RNG of [verts.device]; its meshes live on the CPU, whose generator fork_rng always forks,
    # while asking CUDA for the state of a CPU device fails on a machine without a driver
    real_fork = torch.random.fork_rng

    def fork_rng(devices=None, enabled=True, **kwargs):
        cpu_only = devices is not None and all(torch.device(d).type == "cpu" for d in devices)
        return real_fork(devices=[] if cpu_only else devices, enabled=enabled, **kwargs)

    torch.random.fork_rng = fork_rng
    bench_dir = os.path.join(reference_loader.REFERENCE_ROOT, "actionbench")
    if bench_dir not in sys.path:
        sys.path.insert(0, bench_dir)


def _reference():
    if not reference_loader.available():
        raise SystemExit(f"reference checkout not found at {reference_loader.REFERENCE_ROOT}")
    _install_stubs()
    import benchmark
    import icp
    import sample_mesh
    import sample_point_cloud

    return types.SimpleNamespace(icp=icp, benchmark=benchmark, sample_mesh=sample_mesh, sample_point_cloud=sample_point_cloud)


def _unpack(tf) -> dict:
    """R, T, s of Scale(s).compose(Rotate(R), Translate(T)) as icp.gradient_icp builds it."""
    rot, trans = tf._transforms
    s = torch.diagonal(tf._matrix[0, :3, :3])[None]
    return {"R": rot._matrix[:, :3, :3].clone(), "T": trans._matrix[:, 3, :3].clone(), "s": s.clone()}


def run_icp(pred: torch.Tensor, gt: torch.Tensor, n_iter: int = N_ITER) -> dict:
    """The reference's gradient_icp on the shim, with the best loss after every step (from the losses its
    chamfer_distance calls return)."""
    ref = _reference()
    losses = []
    real = ref.icp.chamfer_distance

    def recording(*args, **kwargs):
        out = real(*args, **kwargs)
        losses.append(out[0].detach().clone())
        return out

    ref.icp.chamfer_distance = recording
    try:
        tf = ref.icp.gradient_icp(pc_pred=pred, pc_gt=gt, lr=0.01, n_iter=n_iter)
    finally:
        ref.icp.chamfer_distance = real
    best, history = float("inf"), []
    for loss in losses:
        m = loss.min()
        if m.item() < best:
            best = m.item()
        history.append(best)
    return {**_unpack(tf), "best_losses": torch.tensor(history, dtype=torch.float64)}


def asymmetric_cloud(n: int, gen: torch.Generator) -> torch.Tensor:
    """Points on an anisotropic ellipsoid with a bump on one side: no symmetry an axis-aligned rotation could match."""
    d = torch.randn(n, 3, generator=gen)
    d = d / d.norm(dim=1, keepdim=True)
    bump = torch.exp(-((d - torch.tensor([0.6, 0.5, 0.62])) ** 2).sum(1) * 8.0)
    return d * torch.tensor([1.0, 0.55, 0.3]) * (1 + 0.6 * bump)[:, None] + torch.tensor([0.1, -0.05, 0.02])


def deforming_mesh(frames: int = 4):
    """A 6 x 12 latitude-longitude sphere, bent progressively along x: one face array, per-frame vertices."""
    lat, lon = 6, 12
    verts = [[0.0, 0.0, 1.0]]
    for i in range(1, lat):
        th = np.pi * i / lat
        verts += [[np.sin(th) * np.cos(2 * np.pi * j / lon), np.sin(th) * np.sin(2 * np.pi * j / lon), np.cos(th)]
                  for j in range(lon)]
    verts.append([0.0, 0.0, -1.0])
    verts = np.array(verts) * np.array([1.0, 0.6, 0.4])
    faces = []
    ring = lambda i, j: 1 + (i - 1) * lon + j % lon  # noqa: E731
    for j in range(lon):
        faces.append([0, ring(1, j), ring(1, j + 1)])
        faces.append([len(verts) - 1, ring(lat - 1, j + 1), ring(lat - 1, j)])
    for i in range(1, lat - 1):
        for j in range(lon):
            faces.append([ring(i, j), ring(i + 1, j), ring(i + 1, j + 1)])
            faces.append([ring(i, j), ring(i + 1, j + 1), ring(i, j + 1)])
    out = []
    for t in range(frames):
        v = verts.copy()
        v[:, 2] += 0.15 * t * v[:, 0] ** 2
        v[:, 1] += 0.05 * t
        out.append(v)
    return np.stack(out), np.array(faces, dtype=np.int64)


def main():
    ref = _reference()
    gen = torch.Generator().manual_seed(7)
    pred = asymmetric_cloud(256, gen)
    R_true = pytorch3d_shim.euler_angles_to_matrix(torch.tensor([[0.4, -1.1, 2.0]]), "XYZ")[0]
    gt = (asymmetric_cloud(240, gen) * torch.tensor([1.2, 0.9, 1.1])) @ R_true + torch.tensor([0.3, -0.2, 0.1])
    icp_out = run_icp(pred, gt)

    verts, faces = deforming_mesh()
    meshes = [_Trimesh(v, faces) for v in verts]
    sample_n = 500
    unsync = ref.sample_mesh.sample_meshes(meshes, n_pts=sample_n, synchronized=False, seed=SEED)
    sync = ref.sample_mesh.sample_meshes(meshes, n_pts=sample_n, synchronized=True, seed=SEED)
    face_idx, _ = ref.sample_mesh.get_baryc_sampling_mesh(ref.sample_mesh.trimesh_to_pytorch3d(meshes[0]), sample_n, SEED)
    sub = ref.sample_point_cloud.sample_point_cloud(unsync, 50, seed=SEED)

    # ground truth for the scores: the same animation under a known similarity transform, densely sampled
    gt_pc = ref.sample_mesh.sample_meshes(meshes, n_pts=3000, synchronized=True, seed=5)
    gt_pc = (gt_pc * torch.tensor([1.1, 0.95, 1.05])) @ R_true + torch.tensor([0.2, 0.1, -0.3])
    scores = ref.benchmark.compute_chamfer_3d_4d(gt_pc, meshes, device="cpu", is_4D=True, n_pts_icp=256,
                                                 n_pts_chamfer=2000, seed=SEED)
    golden = {
        "seed": SEED, "icp_pred": pred, "icp_gt": gt, "icp_n_iter": N_ITER, "icp_R": icp_out["R"], "icp_T": icp_out["T"],
        "icp_s": icp_out["s"], "icp_best_losses": icp_out["best_losses"],
        "canonical": ref.icp.canonical_rotation_matrices(),
        "mesh_vertices": torch.from_numpy(verts), "mesh_faces": torch.from_numpy(faces), "sample_n": sample_n,
        "sample_unsync": unsync, "sample_sync": sync, "sync_face_idx": face_idx[0], "subsample_50": sub,
        "scores_gt": gt_pc, "scores_n_pts_icp": 256, "scores_n_pts_chamfer": 2000,
        "scores": torch.tensor([float(s) for s in scores], dtype=torch.float64),
    }
    torch.save(golden, GOLDEN)
    print("wrote", GOLDEN, "scores", [float(s) for s in scores], "best loss", float(icp_out["best_losses"][-1]))


if __name__ == "__main__":
    if sys.argv[1:2] == ["--rerun-icp"]:   # re-run the stored gradient_icp case and write its result to argv[2]
        g = torch.load(GOLDEN, weights_only=False)
        torch.save(run_icp(g["icp_pred"], g["icp_gt"], n_iter=g["icp_n_iter"]), sys.argv[2])
    else:
        main()
