"""ActionBench's metric kernels bit for bit (-m gpu): amb_nearest_neighbors (csrc/chamfer.cu), amb_icp_chamfer_grad,
amb_icp_transform_points (csrc/icp.cu) against the exact restatements of tests/icp_exact.py, and amb_icp_adam_step against
torch.optim.Adam itself on the CPU and on CUDA.

Shapes sit on and off the kernels' tiles: 128 pred points per pred->gt block, 512 gt points per gt->pred block, 1024
staged points per shared-memory tile, 8 candidates per pred->gt thread and the reference set split over blockIdx.y.
Lattice clouds (coordinates k/8) make ties everywhere, and with power-of-two scales and signed-permutation rotations every
fp32 step is exact, so their sums must also equal an order-free exact sum."""
from __future__ import annotations

import pytest
import torch

import icp_exact as ex
import icp_ref as ref

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _clouds(F: int, P: int, Q: int, seed: int):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(F, P, 3, generator=gen) * torch.tensor([1.0, 0.6, 0.35])
    g = torch.randn(F, Q, 3, generator=gen) * torch.tensor([0.8, 0.7, 0.4]) + 0.05
    return x, g


def _state(F: int, C: int, seed: int):
    """The real canonical R_init (repeated past 24 candidates), parameters near the initial state, R = R_init @ M(d6)."""
    from actionmesh_b200.evaluation import canonical_rotation_matrices

    gen = torch.Generator().manual_seed(seed)
    rot_init = canonical_rotation_matrices()[torch.arange(C) % 24]
    params = ref.initial_state(C)[None].repeat(F, 1, 1) + 0.05 * torch.randn(F, C, 12, generator=gen)
    rot = torch.stack([rot_init @ ref.rot6d_to_matrix(params[f, :, 3:9]) for f in range(F)])
    return rot_init, params, rot


def _check_sums(x, g, rot, params, sums, frames=None):
    for f in range(x.shape[0]) if frames is None else frames:
        want = ex.icp_sums(x[f].to(DEV), g[f].to(DEV), rot[f].to(DEV), params[f].to(DEV))
        ex.assert_bits_equal(sums[f], want, f"frame {f}")


# ---- amb_nearest_neighbors --------------------------------------------------------------------------------------------

def _check_nn(q, r):
    from actionmesh_b200 import ops

    q, r = q.to(DEV), r.to(DEV)
    d, i = ops.nearest_neighbors(q, r)
    d2, want = ex.nearest(q, r)
    assert torch.equal(i.long(), want), int((i.long() != want).sum())
    ex.assert_bits_equal(d, ex.nn_distance(d2), "distance")


@pytest.mark.parametrize("M,N", [(1, 1), (1, 100_003), (129, 1025), (4096, 2048), (23_457, 100_003)])
def test_nearest_neighbors_random(amb_lib, M, N):
    gen = torch.Generator().manual_seed(M + N)
    _check_nn(torch.randn(M, 3, generator=gen), 1.1 * torch.randn(N, 3, generator=gen))


@pytest.mark.parametrize("M,N", [(129, 1025), (4096, 2048), (23_457, 100_003)])
def test_nearest_neighbors_lattice_ties_go_to_the_lowest_index(amb_lib, M, N):
    """Every reference point occurs about 4 times at random indices, and lattice distances tie between distinct points,
    so equal minima straddle the 1024-point tiles and the blockIdx.y chunks."""
    q, r = ex.lattice(M, 1, dup=4) + 1 / 16, ex.lattice(N, 2, dup=4)
    assert torch.unique(r, dim=0).shape[0] <= N // 3
    _check_nn(q, r)


# ---- amb_icp_chamfer_grad --------------------------------------------------------------------------------------------

@pytest.mark.parametrize("F", [1, 3])
@pytest.mark.parametrize("P,Q", [(1, 1), (1, 77), (129, 1), (127, 513), (1025, 1023), (2049, 4097)])
@pytest.mark.parametrize("C", [1, 7, 8, 9, 24, 33])
def test_chamfer_grad_sums(amb_lib, C, P, Q, F):
    from actionmesh_b200 import ops

    x, g = _clouds(F, P, Q, seed=P + 3 * Q + C)
    _, params, rot = _state(F, C, seed=C + F)
    sums = ops.icp_chamfer_grad(x.to(DEV), g.to(DEV), rot.to(DEV), params.to(DEV))
    _check_sums(x, g, rot, params, sums)


def test_chamfer_grad_sums_production_size(amb_lib):
    """16 frames x 24 candidates x 10 000 x 10 000 points, as a 16-frame clip is scored; two frames restated."""
    from actionmesh_b200 import ops

    x, g = _clouds(16, 10_000, 10_000, seed=7)
    _, params, rot = _state(16, 24, seed=8)
    sums = ops.icp_chamfer_grad(x.to(DEV), g.to(DEV), rot.to(DEV), params.to(DEV))
    _check_sums(x, g, rot, params, sums, frames=(0, 15))


@pytest.mark.parametrize("F,P,Q,C", [(2, 2049, 1537, 9), (1, 1025, 4097, 8), (1, 300, 129, 24)])
def test_chamfer_grad_lattice(amb_lib, F, P, Q, C):
    """Exact arithmetic and ties everywhere: the sums equal the restatement and the order-free fsum of the terms."""
    from actionmesh_b200 import ops

    x = torch.stack([ex.lattice(P, 10 + f, dup=4) for f in range(F)])
    g = torch.stack([ex.lattice(Q, 20 + f, dup=4) for f in range(F)])
    rot, params = ex.lattice_transforms(C, C)
    rot, params = rot[None].repeat(F, 1, 1, 1), params[None].repeat(F, 1, 1)
    sums = ops.icp_chamfer_grad(x.to(DEV), g.to(DEV), rot.to(DEV), params.to(DEV))
    _check_sums(x, g, rot, params, sums)
    for f in range(F):
        ex.assert_bits_equal(sums[f].cpu(), ex.fsum_sums(x[f], g[f], rot[f], params[f]), f"fsum, frame {f}")


def test_frames_and_candidates_are_independent(amb_lib):
    from actionmesh_b200 import ops

    x, g = _clouds(3, 1300, 1100, seed=11)
    _, params, rot = _state(3, 24, seed=12)
    x, g, rot, params = x.to(DEV), g.to(DEV), rot.to(DEV), params.to(DEV)
    sums = ops.icp_chamfer_grad(x, g, rot, params)
    for f in range(3):
        one = ops.icp_chamfer_grad(x[f:f + 1].contiguous(), g[f:f + 1].contiguous(), rot[f:f + 1].contiguous(),
                                   params[f:f + 1].contiguous())
        ex.assert_bits_equal(one[0], sums[f], f"frame {f}")
    for n in range(24):
        one = ops.icp_chamfer_grad(x[:1].contiguous(), g[:1].contiguous(), rot[:1, n:n + 1].contiguous(),
                                   params[:1, n:n + 1].contiguous())
        ex.assert_bits_equal(one[0, 0], sums[0, n], f"candidate {n}")


def test_replay_of_the_icp_loop(amb_lib):
    """Ten steps of evaluation.gradient_icp_frames issued by hand: at every step the sums equal the restatement at the
    kernel's own rot and params of that step."""
    from actionmesh_b200 import ops
    from actionmesh_b200.evaluation import canonical_rotation_matrices

    gen = torch.Generator().manual_seed(13)
    shape = torch.randn(1500, 3, generator=gen) * torch.tensor([1.0, 0.55, 0.3])
    R_true = ref.rot6d_to_matrix(torch.tensor([1.0, 0.3, -0.2, -0.1, 1.0, 0.25]))
    gt = (shape[:1300] * torch.tensor([1.1, 0.9, 1.0])) @ R_true + 0.1 + 0.01 * torch.randn(1300, 3, generator=gen)
    x, g = shape[None].to(DEV), gt[None].to(DEV)
    rot_init = canonical_rotation_matrices().to(DEV)
    params = ref.initial_state(24)[None].to(DEV)
    rot = rot_init[None].clone()
    m, v = torch.zeros_like(params), torch.zeros_like(params)
    best = torch.tensor([float("inf")] + [0.0] * 15, device=DEV)[None].contiguous()
    for step in range(1, 11):
        sums = ops.icp_chamfer_grad(x, g, rot, params)
        ex.assert_bits_equal(sums[0], ex.icp_sums(x[0], g[0], rot[0], params[0]), f"step {step}")
        ops.icp_adam_step(sums, rot_init, step, 0.01, params, m, v, rot, best)
    assert float(best[0, 0]) < float(sums[0, :, 0].max())


# ---- amb_icp_adam_step ------------------------------------------------------------------------------------------------

def _run_adam_kernel(sums, rot_init, params, m, v, rot, best, step):
    from actionmesh_b200 import ops

    d = [t.to(DEV).contiguous() for t in (params, m, v, rot, best)]
    ops.icp_adam_step(sums.to(DEV), rot_init.to(DEV), step, 0.01, *d)
    return d


# ---- amb_icp_adam_step against torch.optim.Adam ----------------------------------------------------------------------
#
# The kernel's fp32 update (csrc/icp.cu) is
#   m = fma(0.1, fl(g - m), m),  v = fma(fl(0.001 g), g, fl(0.999 v)),  p = fma(step_size, fl(m / denom), p).
# torch 2.11's Adam orders it differently on its two devices:
#   * CPU, the single-tensor path (the one that wrote tests/golden/actionbench_tiny.pt): m as above,
#     v = fl(fl(fl(0.001 g) g) + fl(0.999 v)), p = fl(p + fl(fl(step_size m) / denom));
#   * CUDA, the foreach path (its default there): m and p as above, v = fma(0.001, fl(g g), fl(0.999 v)).
# So the kernel's m and v are the CPU path's (its v fuses a product the CPU rounds first, which changes the sum only when
# that rounding crosses one of the sum's rounding boundaries: never on these inputs), and its p update is the CUDA
# path's.  The CUDA path's v is the known difference; DESIGN §12 says why the kernel keeps the CPU order.

_SLICES = ((0, 3), (3, 9), (9, 12))        # T, R_6d, s: the three Parameters of icp.py


def _torch_adam(params, m, v, grad, step: int, device: str):
    """torch.optim.Adam(lr=0.01) at its defaults on `device`, state seeded with m, v and step - 1: (C, 12) each -> the new
    (params, m, v) on the GPU."""
    ps = [torch.nn.Parameter(params[:, a:b].to(device).clone()) for a, b in _SLICES]
    opt = torch.optim.Adam(ps, lr=0.01)
    for p, (a, b) in zip(ps, _SLICES):
        p.grad = grad[:, a:b].to(device).clone()
        opt.state[p] = {"step": torch.tensor(float(step - 1)), "exp_avg": m[:, a:b].to(device).clone(),
                        "exp_avg_sq": v[:, a:b].to(device).clone()}
    opt.step()
    cat = lambda key: torch.cat([opt.state[p][key] for p in ps], 1).to(DEV)
    return torch.cat([p.detach() for p in ps], 1).to(DEV), cat("exp_avg"), cat("exp_avg_sq")


def _check_adam_against_torch(got, params, m, v, grad, step, mask=None):
    """The kernel's (params, m, v) of one frame against torch.optim.Adam, at the elements of `mask`:
      * CPU Adam: m and v bit for bit; params within the CPU's two extra roundings of the step (<= 3u of it) plus one ulp;
      * CUDA Adam: m bit for bit, and params bit for bit wherever the kernel's v equals CUDA's."""
    mask = torch.ones_like(got[0], dtype=torch.bool) if mask is None else mask
    (p_k, m_k, v_k), p64 = got, params.double().to(DEV)
    p_c, m_c, v_c = _torch_adam(params, m, v, grad, step, "cpu")
    ex.assert_bits_equal(m_k[mask], m_c[mask], f"m against CPU Adam, step {step}")
    ex.assert_bits_equal(v_k[mask], v_c[mask], f"v against CPU Adam, step {step}")
    inc = (p_c.double() - p64).abs()
    ulp = torch.nextafter(p_c.abs(), torch.tensor(float("inf"), device=DEV)) - p_c.abs()
    assert bool(((p_k - p_c).abs() <= ulp + 2.0 ** -22 * inc)[mask].all()), f"params against CPU Adam, step {step}"
    p_g, m_g, v_g = _torch_adam(params, m, v, grad, step, "cuda")
    ex.assert_bits_equal(m_k[mask], m_g[mask], f"m against CUDA Adam, step {step}")
    same_v = mask & (ex.bits(v_k) == ex.bits(v_g))
    ex.assert_bits_equal(p_k[same_v], p_g[same_v], f"params against CUDA Adam where v agrees, step {step}")


def _exact_case(step: int):
    """R_init = I, d6 = (2^a, 0, 0, 0, 2^b, 0), dyadic s and sums, C = 32: every step of the closed-form backward is exact,
    so the fp32 gradient the kernel hands to Adam is known exactly.  For t > 1, v is of the size 0.001 g g (as after the
    gradient has grown), so that the two orders of v differ at every step."""
    F, C = 2, 32
    gen = torch.Generator().manual_seed(step)
    rot_init = torch.eye(3).repeat(C, 1, 1)
    params = torch.randn(F, C, 12, generator=gen)
    params[..., 3:9] = 0
    params[..., 3] = torch.exp2(torch.randint(-2, 3, (F, C), generator=gen).float())
    params[..., 7] = torch.exp2(torch.randint(-2, 3, (F, C), generator=gen).float())
    params[..., 9:] = torch.randint(1, 16, (F, C, 3), generator=gen).float() / 8
    rot = torch.eye(3).repeat(F, C, 1, 1)
    sums = torch.randint(-2 ** 12, 2 ** 12, (F, C, 13), generator=gen).double() / 2 ** 14
    sums[..., 0] = sums[..., 0].abs()
    grads = torch.stack([ref.param_grads(sums[f], rot_init, rot[f], params[f]) for f in range(F)])
    assert torch.equal(grads.float().double(), grads)            # the premise: an exact fp32 gradient
    m = (1 - 0.9 ** (step - 1)) * grads.float() * (0.5 + torch.rand(F, C, 12, generator=gen))
    v = (step > 1) * 0.001 * grads.float() ** 2 * (0.5 + torch.rand(F, C, 12, generator=gen))
    best = torch.zeros(F, 16)
    best[:, 0] = float("inf")
    got = _run_adam_kernel(sums, rot_init, params, m, v, rot, best, step)
    return got, params, m, v, grads.float()


@pytest.mark.parametrize("step", [1, 2, 7, 200])
def test_adam_step_exact_gradients(amb_lib, step):
    got, params, m, v, grads = _exact_case(step)
    for f in range(params.shape[0]):
        _check_adam_against_torch([t[f] for t in got[:3]], params[f], m[f], v[f], grads[f], step)


@pytest.mark.xfail(strict=True, raises=AssertionError, reason="the kernel's v = fma(fl(0.001 g), g, fl(0.999 v)) keeps the order of torch's CPU "
                                       "Adam; torch's CUDA Adam computes fma(0.001, fl(g g), fl(0.999 v)), an ulp apart "
                                       "in about a fifth of the elements at t = 1 (DESIGN §12)")
@pytest.mark.parametrize("step", [1, 2, 7, 200])
def test_adam_step_equals_torch_cuda_adam(amb_lib, step):
    """The whole update against torch's CUDA Adam (foreach, the default on CUDA) bit for bit.  Expected to fail until the
    kernel takes the CUDA order of v; strict, so that it reports when it starts to pass."""
    got, params, m, v, grads = _exact_case(step)
    for f in range(params.shape[0]):
        want = _torch_adam(params[f], m[f], v[f], grads[f], step, "cuda")
        for name, a, b in zip(("params", "m", "v"), [t[f] for t in got[:3]], want):
            ex.assert_bits_equal(a, b, f"{name}, step {step}")


def _rot_bound(d6: torch.Tensor, rot_init: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """R_init @ rotation_6d_to_matrix(d6) in fp64 and a first-order bound on the kernel's fp32 error per entry, carried
    through the kernel's operations (normalize, Gram-Schmidt, cross product, the 3-term product; each rounding <= u of
    its result, contraction only removes roundings), with 1 % for second-order terms."""
    u = 2.0 ** -24
    d6, ri = d6.double(), rot_init.double()
    a1, a2 = d6[:, :3], d6[:, 3:]
    sq = (a1 * a1).sum(1, keepdim=True)
    n1 = sq.sqrt()
    e_n1 = 3 * u * sq / (2 * n1) + u * n1
    b1 = a1 / n1
    e_b1 = a1.abs() * e_n1 / n1 ** 2 + u * b1.abs()
    dot = (b1 * a2).sum(1, keepdim=True)
    e_dot = (e_b1 * a2.abs()).sum(1, keepdim=True) + 3 * u * (b1 * a2).abs().sum(1, keepdim=True)
    w = a2 - dot * b1
    e_w = e_dot * b1.abs() + dot.abs() * e_b1 + u * (dot * b1).abs() + u * w.abs()
    sq2 = (w * w).sum(1, keepdim=True)
    n2 = sq2.sqrt()
    e_n2 = ((2 * w.abs() * e_w).sum(1, keepdim=True) + 3 * u * sq2) / (2 * n2) + u * n2
    b2 = w / n2
    e_b2 = e_w / n2 + w.abs() * e_n2 / n2 ** 2 + u * b2.abs()
    b3, e_b3 = torch.empty_like(b1), torch.empty_like(b1)
    for l, (i, j) in enumerate(((1, 2), (2, 0), (0, 1))):
        p, q = b1[:, i] * b2[:, j], b1[:, j] * b2[:, i]
        b3[:, l] = p - q
        e_b3[:, l] = (e_b1[:, i] * b2[:, j].abs() + b1[:, i].abs() * e_b2[:, j] + e_b1[:, j] * b2[:, i].abs()
                      + b1[:, j].abs() * e_b2[:, i] + u * (p.abs() + q.abs() + b3[:, l].abs()))
    M, e_M = torch.stack((b1, b2, b3), 1), torch.stack((e_b1, e_b2, e_b3), 1)
    R = (ri[:, :, :, None] * M[:, None]).sum(2)
    e_R = (ri.abs()[:, :, :, None] * e_M[:, None]).sum(2) + 5 * u * (ri.abs()[:, :, :, None] * M.abs()[:, None]).sum(2)
    return R, 1.01 * e_R


@pytest.mark.parametrize("step", [1, 4, 200])
def test_adam_step_random_state(amb_lib, step):
    """Real R_init and kernel sums.  The kernel's fp64 backward may round differently from icp_ref's (a few fp64 ulps,
    more where the 6D backward cancels), so only elements whose fp64 gradient lies more than 2^-36 (relative) from an fp32
    rounding boundary are compared; at least 99 % are.  (At 2^-29 about 3 % of the elements drop out: the boundary
    distance is spread over half an fp32 ulp, 2^-25 relative.)
    Also: the best-candidate bookkeeping, and R of the new parameters within its derived per-entry bound."""
    from actionmesh_b200 import ops

    F, C = 2, 24
    x, g = _clouds(F, 200, 180, seed=1)
    rot_init, params, rot = _state(F, C, seed=2)
    gen = torch.Generator().manual_seed(3)
    m = 1e-3 * torch.randn(F, C, 12, generator=gen)
    v = 1e-6 * torch.rand(F, C, 12, generator=gen)
    best = torch.zeros(F, 16)
    best[:, 0] = float("inf")
    best[1, 0] = 0.0                          # frame 1: nothing beats the best so far
    sums = ops.icp_chamfer_grad(x.to(DEV), g.to(DEV), rot.to(DEV), params.to(DEV)).cpu()
    low = float(sums[0, :, 0].min()) * 0.5    # an exact tie between candidates 3 and 5, below every other candidate
    sums[0, 3, 0] = low
    sums[0, 5, 0] = low
    d_params, d_m, d_v, d_rot, d_best = _run_adam_kernel(sums, rot_init, params, m, v, rot, best, step)
    for f in range(F):
        grad = ref.param_grads(sums[f], rot_init, rot[f], params[f])
        g32 = grad.float()
        lo = (g32.double() + torch.nextafter(g32, torch.tensor(-float("inf"))).double()) / 2
        hi = (g32.double() + torch.nextafter(g32, torch.tensor(float("inf"))).double()) / 2
        margin = torch.minimum((grad - lo).abs(), (hi - grad).abs()) / grad.abs()
        mask = (margin > 2.0 ** -36) & (grad != 0)
        assert float(mask.double().mean()) >= 0.99, float(mask.double().mean())
        _check_adam_against_torch([d_params[f], d_m[f], d_v[f]], params[f], m[f], v[f], g32, step, mask=mask.to(DEV))
        R, bound = _rot_bound(d_params[f, :, 3:9].cpu(), rot_init)
        err = (d_rot[f].cpu().double() - R).abs()
        assert bool((err <= bound).all()), float((err / bound).max())
        want = ref.best_update(sums[f, :, 0].float(), best[f], rot[f], d_params[f].cpu())
        assert torch.equal(d_best[f].cpu(), want), f
    assert torch.equal(d_best[0, 1:10].cpu(), rot[0, 3].reshape(9))    # the tie went to the lower index, R before the step
    assert torch.equal(d_best[1].cpu(), best[1])


# ---- amb_icp_transform_points ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("per_frame", [True, False])
@pytest.mark.parametrize("N", [1, 1000, 70_001])
def test_transform_points(amb_lib, per_frame, N):
    from actionmesh_b200 import ops

    gen = torch.Generator().manual_seed(N)
    p = torch.randn(3, N, 3, generator=gen)
    k = 3 if per_frame else 1
    R = ref.rot6d_to_matrix(torch.randn(k, 6, generator=gen))
    tf = torch.cat([R.reshape(k, 9), torch.randn(k, 3, generator=gen), 0.5 + torch.rand(k, 3, generator=gen)], 1)
    got = ops.icp_transform_points(p.to(DEV), tf.to(DEV))
    ex.assert_bits_equal(got, ex.transform_points(p.to(DEV), tf.to(DEV)), "transform_points")
