"""ActionBench gradient ICP on the host: the closed-form math of csrc/icp.cu (tests/icp_ref.py) against torch autograd and
torch.optim.Adam, the reference's best-candidate bookkeeping, the canonical rotations and mesh sampling against the golden
from the reference's own code (tools/gen_actionbench_golden.py), the ABI's argument checks, and the dataset driver."""
from __future__ import annotations

import csv
import json
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import icp_ref as ref
from conftest import ROOT, load_golden

sys.path.insert(0, os.path.join(ROOT, "tools"))

GOLDEN_FILE = "actionbench_tiny.pt"


def _rot_init():
    from actionmesh_b200.evaluation import canonical_rotation_matrices

    return canonical_rotation_matrices()


def _case(seed: int, P: int, Q: int, C: int = 24, degenerate: bool = False):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(P, 3, generator=gen, dtype=torch.float64) * torch.tensor([1.0, 0.6, 0.3], dtype=torch.float64)
    g = torch.randn(Q, 3, generator=gen, dtype=torch.float64) * torch.tensor([0.9, 0.7, 0.4], dtype=torch.float64) + 0.1
    params = ref.initial_state(C).double()
    params += 0.3 * torch.randn(C, 12, generator=gen, dtype=torch.float64)
    params[:, 9:] = 0.5 + torch.rand(C, 3, generator=gen, dtype=torch.float64)
    if degenerate:   # a2 nearly parallel to a1, and a tiny a1
        params[:C // 2, 6:9] = params[:C // 2, 3:6] * 1.5 + 1e-4 * torch.randn(C // 2, 3, generator=gen, dtype=torch.float64)
        params[C // 2:, 3:6] *= 1e-3
    return x, g, params


@pytest.mark.parametrize("degenerate", [False, True])
def test_closed_form_gradient_matches_autograd(degenerate):
    """The 12 sums, the 1/C scaling and the 6D backward equal autograd on the reference loss in fp64 to 1e-10."""
    rot_init = _rot_init().double()
    x, g, params = _case(3 + degenerate, 37, 29, degenerate=degenerate)
    p = params.clone().requires_grad_(True)
    R = rot_init @ ref.rot6d_to_matrix(p[:, 3:9])
    loss = ref.chamfer_loss(ref.transform(x, R, p[:, 9:], p[:, :3]), g)
    loss.mean().backward()
    sums = ref.chamfer_sums(x, g, R.detach(), params[:, 9:], params[:, :3])
    assert torch.allclose(sums[:, 0], loss.detach(), rtol=1e-13, atol=0)
    got = ref.param_grads(sums, rot_init, R.detach(), params)
    err = (got - p.grad).norm() / p.grad.norm()
    assert err <= 1e-10, err
    for n in range(24):   # per candidate too, so a small candidate cannot hide behind a large one
        assert (got[n] - p.grad[n]).norm() <= 1e-10 * p.grad[n].norm() + 1e-300


def test_adam_matches_torch_optim():
    gen = torch.Generator().manual_seed(11)
    p0 = torch.randn(24, 12, generator=gen)
    p = torch.nn.Parameter(p0.clone())
    opt = torch.optim.Adam([p], lr=0.01)
    mine, m, v = p0.clone(), torch.zeros_like(p0), torch.zeros_like(p0)
    for step in range(1, 4):
        grad = torch.randn(24, 12, generator=gen) * (10.0 ** -step)
        p.grad = grad.clone()
        opt.step()
        mine, m, v = ref.adam_step(mine, m, v, grad, step, 0.01)
        assert torch.allclose(mine, p.detach(), rtol=1e-6, atol=1e-7)
        assert torch.allclose(m, opt.state[p]["exp_avg"], rtol=1e-6, atol=0)
        assert torch.allclose(v, opt.state[p]["exp_avg_sq"], rtol=1e-6, atol=0)


def test_best_tracking_quirks():
    R_pre = torch.arange(3 * 9, dtype=torch.float32).reshape(3, 3, 3)
    post = torch.arange(3 * 12, dtype=torch.float32).reshape(3, 12) + 100
    best = torch.zeros(16)
    best[0] = float("inf")
    b1 = ref.best_update(torch.tensor([2.0, 1.0, 1.0]), best, R_pre, post)
    assert b1[0] == 1.0 and torch.equal(b1[1:10], R_pre[1].reshape(9))       # lowest index among equal minima
    assert torch.equal(b1[10:13], post[1, :3]) and torch.equal(b1[13:], post[1, 9:])   # T and s after the step
    assert torch.equal(ref.best_update(torch.tensor([1.0, 3.0, 4.0]), b1, R_pre, post), b1)   # not strictly below
    assert torch.equal(ref.best_update(torch.tensor([0.5, float("nan"), 4.0]), b1, R_pre, post), b1)   # NaN: min is NaN
    assert ref.best_update(torch.tensor([0.5, 0.25, 4.0]), b1, R_pre, post)[0] == 0.25


def test_reference_restatement_runs_the_quirks():
    """The reference loop restated in torch (tools/actionbench_bench.eager_gradient_icp) records R before the step and T, s
    after it, and matches icp_ref step by step."""
    from actionbench_bench import eager_gradient_icp

    x, g, _ = _case(5, 20, 17)
    x, g = x.float(), g.float()
    best, history = eager_gradient_icp(x, g, n_iter=3, lr=0.01, with_history=True)
    rot_init = _rot_init()
    params, m, v = ref.initial_state(24), torch.zeros(24, 12), torch.zeros(24, 12)
    mine = torch.zeros(16)
    mine[0] = float("inf")
    for step in range(1, 4):
        R = rot_init @ ref.rot6d_to_matrix(params[:, 3:9])
        sums = ref.chamfer_sums(x.double(), g.double(), R.double(), params[:, 9:].double(), params[:, :3].double())
        grads = ref.param_grads(sums, rot_init, R, params)
        params, m, v = ref.adam_step(params, m, v, grads, step, 0.01)
        mine = ref.best_update(sums[:, 0].float(), mine, R, params)
        assert abs(float(history[step - 1]) - float(mine[0])) <= 1e-5 * float(mine[0])
    assert torch.allclose(best, mine, rtol=1e-4, atol=1e-6)


@pytest.fixture(scope="module")
def golden():
    return load_golden(GOLDEN_FILE)


def test_canonical_rotations_equal_the_reference(golden):
    got = _rot_init()
    assert got.dtype == torch.float32 and torch.equal(got, golden["canonical"])
    off = got.abs()[(got.abs() < 1e-6) & (got != 0)]
    assert off.numel() and float(off.max()) < 1e-7       # the fp32 cos(pi/2) residues are kept


def _golden_meshes(golden):
    return [SimpleNamespace(vertices=v.numpy(), faces=golden["mesh_faces"].numpy()) for v in golden["mesh_vertices"]]


@pytest.mark.parametrize("synchronized", [False, True])
def test_sample_meshes_matches_the_reference(golden, synchronized):
    from actionmesh_b200.evaluation import sample_meshes

    key = "sample_sync" if synchronized else "sample_unsync"
    got = sample_meshes(_golden_meshes(golden), n_pts=golden["sample_n"], synchronized=synchronized, seed=golden["seed"])
    want = golden[key]
    assert got.dtype == torch.float32 and got.shape == want.shape
    assert float((got - want).abs().max()) <= 1e-6


def test_synchronized_faces_match_the_reference(golden):
    from actionmesh_b200.evaluation import _synchronized_sampling

    m = _golden_meshes(golden)[0]
    face_idx, _ = _synchronized_sampling(np.asarray(m.vertices), m.faces, golden["sample_n"], golden["seed"])
    assert np.array_equal(face_idx, golden["sync_face_idx"].numpy())


def test_sample_point_cloud_matches_the_reference(golden):
    from actionmesh_b200.evaluation import sample_point_cloud

    assert torch.equal(sample_point_cloud(golden["sample_unsync"], 50, seed=golden["seed"]), golden["subsample_50"])


def test_shim_reproduces_the_golden(golden, tmp_path):
    """The reference's gradient_icp on oracle/pytorch3d_shim.py, re-run in a fresh interpreter (the generator installs
    module stubs), gives the stored per-step best losses and result bit for bit.  Needs the reference checkout."""
    from oracle import reference_loader

    if not reference_loader.available():
        pytest.skip("the reference checkout is not available")
    out = tmp_path / "icp.pt"
    subprocess.run([sys.executable, os.path.join(ROOT, "tools", "gen_actionbench_golden.py"), "--rerun-icp", str(out)],
                   check=True, cwd=ROOT, timeout=600)
    got = torch.load(out, weights_only=False)
    assert torch.equal(got["best_losses"], golden["icp_best_losses"])
    for k in ("R", "T", "s"):
        assert torch.equal(got[k], golden[f"icp_{k}"]), k


def test_icp_abi_refuses_bad_arguments(amb_lib):
    P = 16
    err = lambda: amb_lib.amb_last_error().decode()  # noqa: E731
    assert amb_lib.amb_icp_chamfer_grad(None, P, 1, 24, 8, 8, P, P, P, P, None) < 0 and "null pointer" in err()
    assert amb_lib.amb_icp_chamfer_grad(P, P, 1, 24, 0, 8, P, P, P, P, None) < 0 and "bad sizes" in err()
    assert amb_lib.amb_icp_chamfer_grad(P, P, 1, 0, 8, 8, P, P, P, P, None) < 0 and "bad sizes" in err()
    assert amb_lib.amb_icp_chamfer_grad(P, P, 0, 24, 8, 8, P, P, P, P, None) < 0 and "bad sizes" in err()
    assert amb_lib.amb_icp_adam_step(P, P, 1, 1025, 0.0, 1.0, P, P, P, P, P, None) < 0 and "bad sizes" in err()
    assert amb_lib.amb_icp_adam_step(P, None, 1, 24, 0.0, 1.0, P, P, P, P, P, None) < 0 and "null pointer" in err()
    assert amb_lib.amb_icp_transform_points(P, 1, 8, None, 0, P, None) < 0 and "null pointer" in err()
    import ctypes

    n = ctypes.c_int64()
    assert amb_lib.amb_icp_scratch_doubles(2, 24, 10_000, 10_000, ctypes.byref(n)) == 0
    assert n.value == 2 * 24 * (79 + 20) * 13


def test_icp_ops_refuse_cpu_tensors():
    from actionmesh_b200 import AmbError, evaluation, ops

    x = torch.zeros(1, 8, 3)
    with pytest.raises(AmbError):
        ops.icp_chamfer_grad(x, x, torch.zeros(1, 24, 3, 3), torch.zeros(1, 24, 12))
    with pytest.raises(AmbError):
        evaluation.gradient_icp(x[0], x[0])


# ---- dataset driver (tools/actionbench_eval.py) ----------------------------------------------------------------------


def _tree(tmp_path, uids, n_meshes, n_frames=3):
    gt_root, pred_root = tmp_path / "gt", tmp_path / "pred"
    for uid in uids:
        (gt_root / uid).mkdir(parents=True)
        np.save(gt_root / uid / "surfaces.npy", np.zeros((n_frames, 10, 6), dtype=np.float64) + 0.5)
        (pred_root / uid).mkdir(parents=True)
        for k in range(n_meshes):
            (pred_root / uid / f"mesh_{k}.glb").write_bytes(b"")
    return gt_root, pred_root


def test_natural_sort():
    import actionbench_eval as ev

    names = ["mesh_10.glb", "mesh_2.glb", "mesh_1.glb", "mesh_001a.glb"]
    assert ev.natural_sorted(names) == ["mesh_1.glb", "mesh_001a.glb", "mesh_2.glb", "mesh_10.glb"]


def test_dataset_driver(tmp_path):
    import actionbench_eval as ev

    gt_root, pred_root = _tree(tmp_path, ["b", "a"], n_meshes=12)
    _tree(tmp_path / "c", ["c"], n_meshes=2)                # 3 GT frames, only 2 predicted meshes
    _tree(tmp_path / "e", ["e"], n_meshes=0)                # GT without any prediction: not a common uid
    for side in ("gt", "pred"):
        for uid in ("c", "e"):
            src = tmp_path / uid / side / uid
            if src.exists():
                os.rename(src, (gt_root if side == "gt" else pred_root) / uid)
    seen = {}

    def scorer(gt_pc, mesh_paths):
        uid = os.path.basename(os.path.dirname(mesh_paths[0]))
        seen[uid] = (gt_pc, mesh_paths)
        return 0.1, 0.2, 0.3

    out = tmp_path / "res.csv"
    rows = ev.evaluate_dataset(str(gt_root), str(pred_root), str(out), scorer=scorer)
    assert [r["uid"] for r in rows] == ["a", "b", "c"]
    gt_pc, paths = seen["a"]
    assert gt_pc.dtype == np.float32 and gt_pc.shape == (3, 10, 3)
    assert [os.path.basename(p) for p in paths] == ["mesh_0.glb", "mesh_1.glb", "mesh_2.glb"]   # natural order, truncated
    assert rows[2]["status"] == "error" and "Not enough meshes" in rows[2]["error_message"] and rows[0]["cd_3d"] == 0.1
    with open(out) as f:
        got = list(csv.DictReader(f))
    assert [r["uid"] for r in got] == ["a", "b", "c"] and list(got[0]) == ev.COLUMNS
    summary = json.load(open(tmp_path / "res.summary.json"))
    assert summary["n_success"] == 2 and summary["n_failed"] == 1 and abs(summary["cd_4d_mean"] - 0.2) < 1e-12

    # resume: rows that succeeded are kept, the failed uid is retried
    seen.clear()
    rows = ev.evaluate_dataset(str(gt_root), str(pred_root), str(out), scorer=scorer)
    assert list(seen) == [] and [r["status"] for r in rows] == ["success", "success", "error"]
    for k in (2, 3):
        (pred_root / "c" / f"mesh_{k}.glb").write_bytes(b"")
    rows = ev.evaluate_dataset(str(gt_root), str(pred_root), str(out), scorer=scorer)
    assert list(seen) == ["c"] and [r["status"] for r in rows] == ["success"] * 3


def test_missing_trimesh_is_a_clear_error(monkeypatch):
    import actionbench_eval as ev

    monkeypatch.setitem(sys.modules, "trimesh", None)
    with pytest.raises(RuntimeError, match="needs trimesh"):
        ev.load_meshes(["x.glb"])
