"""ActionBench gradient ICP on the GPU (csrc/icp.cu, evaluation.gradient_icp / compute_chamfer_3d_4d).

One step against the fp64 restatement of tests/icp_ref.py at several sizes (P != Q, sizes off the tiles, P = 1 and the
production 10 000 x 10 000 at F = 16), the Adam step against icp_ref on the same sums, full runs against the golden written
by the reference's own code (tools/gen_actionbench_golden.py), a known answer, determinism and argument errors."""
from __future__ import annotations

import pytest
import torch

import icp_ref as ref
from conftest import load_golden

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _state(F: int, C: int, seed: int):
    from actionmesh_b200.evaluation import canonical_rotation_matrices

    gen = torch.Generator().manual_seed(seed)
    rot_init = canonical_rotation_matrices()
    params = ref.initial_state(C)[None].repeat(F, 1, 1)
    params += 0.05 * torch.randn(F, C, 12, generator=gen)
    rot = torch.stack([rot_init @ ref.rot6d_to_matrix(params[f, :, 3:9]) for f in range(F)])
    return rot_init, params, rot


def _clouds(F: int, P: int, Q: int, seed: int):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(F, P, 3, generator=gen) * torch.tensor([1.0, 0.6, 0.35])
    g = torch.randn(F, Q, 3, generator=gen) * torch.tensor([0.8, 0.7, 0.4]) + 0.05
    return x, g


def _ref_sums_fp64(x, g, rot, params):
    """(C, 13) fp64 sums with fp64 nearest neighbours, evaluated on the GPU candidate by candidate."""
    x, g = x.to(DEV, torch.float64), g.to(DEV, torch.float64)
    out = []
    for n in range(rot.shape[0]):
        R, s, T = rot[n:n + 1].to(DEV, torch.float64), params[n:n + 1, 9:].to(DEV, torch.float64), \
            params[n:n + 1, :3].to(DEV, torch.float64)
        y = ref.transform(x, R, s, T)[0]
        d = torch.cdist(y, g, compute_mode="donot_use_mm_for_euclid_dist") ** 2
        a, b = d.argmin(1), d.argmin(0)
        out.append(ref.chamfer_sums(x, g, R, s, T, a=a[None], b=b[None])[0].cpu())
        del d
    return torch.stack(out)


@pytest.mark.parametrize("F,P,Q,check", [(2, 300, 257, 2), (2, 1, 77, 2), (2, 1000, 1531, 2), (2, 129, 1, 2),
                                         (16, 10_000, 10_000, 2)])
def test_one_step_matches_fp64(amb_lib, F, P, Q, check):
    from actionmesh_b200 import ops

    C = 24
    x, g = _clouds(F, P, Q, seed=P + Q)
    rot_init, params, rot = _state(F, C, seed=F + P)
    sums = ops.icp_chamfer_grad(x.to(DEV), g.to(DEV), rot.to(DEV), params.to(DEV)).cpu()
    for f in range(check):
        want = _ref_sums_fp64(x[f], g[f], rot[f], params[f])
        assert torch.allclose(sums[f, :, 0], want[:, 0], rtol=1e-5, atol=0), (f, sums[f, :, 0], want[:, 0])
        err = (sums[f, :, 1:] - want[:, 1:]).norm(dim=1) / want[:, 1:].norm(dim=1)
        assert float(err.max()) <= 1e-4, (f, err)


def test_adam_step_matches_icp_ref(amb_lib):
    from actionmesh_b200 import ops

    F, C, P, Q = 2, 24, 200, 180
    x, g = _clouds(F, P, Q, seed=1)
    rot_init, params, rot = _state(F, C, seed=2)
    gen = torch.Generator().manual_seed(3)
    m = 1e-3 * torch.randn(F, C, 12, generator=gen)
    v = 1e-6 * torch.rand(F, C, 12, generator=gen)
    best = torch.zeros(F, 16)
    best[:, 0] = float("inf")
    best[1, 0] = 0.0                          # frame 1: nothing beats the best so far
    d_params, d_m, d_v, d_rot, d_best = (t.to(DEV).contiguous() for t in (params, m, v, rot, best))
    sums = ops.icp_chamfer_grad(x.to(DEV), g.to(DEV), d_rot, d_params)
    low = float(sums[0, :, 0].min()) * 0.5    # an exact tie between candidates 3 and 5, below every other candidate
    sums[0, 3, 0] = low
    sums[0, 5, 0] = low
    step = 4
    ops.icp_adam_step(sums, rot_init.to(DEV), step, 0.01, d_params, d_m, d_v, d_rot, d_best)
    sums = sums.cpu()
    for f in range(F):
        grads = ref.param_grads(sums[f], rot_init, rot[f], params[f])
        p_new, m_new, v_new = ref.adam_step(params[f], m[f], v[f], grads, step, 0.01)
        assert torch.allclose(d_params[f].cpu(), p_new, rtol=1e-6, atol=1e-7)
        assert torch.allclose(d_m[f].cpu(), m_new, rtol=1e-6, atol=1e-12)
        assert torch.allclose(d_v[f].cpu(), v_new, rtol=1e-6, atol=1e-15)
        assert torch.allclose(d_rot[f].cpu(), rot_init @ ref.rot6d_to_matrix(p_new[:, 3:9]), rtol=0, atol=1e-6)
        want = ref.best_update(sums[f, :, 0].float(), best[f], rot[f], d_params[f].cpu())
        assert torch.equal(d_best[f].cpu(), want), f
    assert torch.equal(d_best[0, 1:10].cpu(), rot[0, 3].reshape(9))    # the tie went to the lower index, R before the step
    assert torch.equal(d_best[1].cpu(), best[1])


@pytest.fixture(scope="module")
def golden():
    return load_golden("actionbench_tiny.pt")


def _bbox_diag(p: torch.Tensor) -> float:
    return float((p.reshape(-1, 3).max(0).values - p.reshape(-1, 3).min(0).values).norm())


def test_gradient_icp_matches_the_reference(amb_lib, golden):
    from actionmesh_b200.evaluation import gradient_icp

    pred, gt = golden["icp_pred"], golden["icp_gt"]
    tf = gradient_icp(pred.to(DEV), gt.to(DEV), n_iter=golden["icp_n_iter"])
    want_loss = float(golden["icp_best_losses"][-1])
    assert abs(float(tf.loss[0]) - want_loss) <= 1e-3 * want_loss
    want = (pred * golden["icp_s"]) @ golden["icp_R"][0] + golden["icp_T"]
    got = tf.transform_points(pred.to(DEV)).cpu()
    assert float((got - want).norm(dim=1).max()) <= 1e-3 * _bbox_diag(gt)


def test_chamfer_3d_4d_matches_the_reference(amb_lib, golden):
    from types import SimpleNamespace

    from actionmesh_b200.evaluation import compute_chamfer_3d_4d

    meshes = [SimpleNamespace(vertices=v.numpy(), faces=golden["mesh_faces"].numpy()) for v in golden["mesh_vertices"]]
    got = compute_chamfer_3d_4d(golden["scores_gt"], meshes, device=DEV, is_4D=True,
                                n_pts_icp=golden["scores_n_pts_icp"], n_pts_chamfer=golden["scores_n_pts_chamfer"],
                                seed=golden["seed"])
    for g, w in zip(got, golden["scores"].tolist()):
        assert abs(g - w) <= 1e-3 * abs(w), (got, golden["scores"])


def test_known_answer(amb_lib):
    """An asymmetric shape under a rotation, an anisotropic scale and a translation, plus noise, is recovered to the noise."""
    from actionmesh_b200.evaluation import gradient_icp

    gen = torch.Generator().manual_seed(21)
    d = torch.randn(3000, 3, generator=gen)
    d = d / d.norm(dim=1, keepdim=True)
    bump = torch.exp(-((d - torch.tensor([0.6, 0.5, 0.62])) ** 2).sum(1) * 8.0)
    shape = d * torch.tensor([1.0, 0.55, 0.3]) * (1 + 0.6 * bump)[:, None]
    R_true = ref.rot6d_to_matrix(torch.tensor([1.0, 0.25, -0.15, -0.2, 1.0, 0.3]))
    s_true, T_true, sigma = torch.tensor([1.15, 0.9, 1.05]), torch.tensor([0.2, -0.1, 0.15]), 2e-3
    gt = (shape * s_true) @ R_true + T_true + sigma * torch.randn(3000, 3, generator=gen)
    tf = gradient_icp(shape.to(DEV), gt.to(DEV))
    aligned = tf.transform_points(shape.to(DEV)).cpu()
    rms = float(((aligned - gt) ** 2).sum(1).mean().sqrt())
    assert rms <= 4 * sigma * 3 ** 0.5, rms


def test_deterministic_and_unified_equals_frame_zero(amb_lib):
    from actionmesh_b200.evaluation import gradient_icp, gradient_icp_frames

    x, g = _clouds(3, 700, 650, seed=9)
    x, g = x.to(DEV), g.to(DEV)
    a = gradient_icp_frames(x, g, n_iter=30)
    b = gradient_icp_frames(x, g, n_iter=30)
    assert torch.equal(a.packed, b.packed)
    u = gradient_icp(x[0], g[0], n_iter=30)
    assert torch.equal(u.packed[0], a.packed[0])


def test_errors(amb_lib):
    from actionmesh_b200 import AmbError, ops
    from actionmesh_b200.evaluation import gradient_icp

    x = torch.randn(50, 3)
    with pytest.raises(AmbError):
        gradient_icp(x, x)
    with pytest.raises(AmbError):
        gradient_icp(x.to(DEV, torch.float64), x.to(DEV, torch.float64))
    with pytest.raises(AmbError):
        gradient_icp(torch.empty(0, 3, device=DEV), x.to(DEV))
    rot_init, params, rot = _state(1, 24, 0)
    with pytest.raises(AmbError):
        ops.icp_chamfer_grad(x[None].to(DEV), x[None].to(DEV), rot.to(DEV), params.double().to(DEV))
