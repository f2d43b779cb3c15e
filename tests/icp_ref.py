"""Restatement in torch of the gradient-ICP kernels' closed-form math (csrc/icp.cu), for the ICP tests.

Not collected by pytest.  Everything takes and returns CPU tensors:
  * `chamfer_loss` — the reference loss (pytorch3d chamfer_distance semantics) by brute force, differentiable;
  * `chamfer_sums` — the loss and the 12 gradient sums t, A of every candidate, from explicit nearest-neighbour choices;
  * `rot6d_to_matrix` / `rot6d_backward` — pytorch3d's 6D rotation and the closed-form backward the kernel uses;
  * `param_grads` — dL/d(T, d6, s) of loss.mean() over the candidates from the sums;
  * `adam_step` — torch.optim.Adam's update at its defaults, fp32, to a few ulps;
  * `best_update` — icp.py:99-106's bookkeeping (pre-step R, post-step T and s; NaN anywhere records nothing).
"""
from __future__ import annotations

import torch


def transform(x: torch.Tensor, R: torch.Tensor, s: torch.Tensor, T: torch.Tensor) -> torch.Tensor:
    """x (P, 3), R (C, 3, 3), s (C, 3), T (C, 3) -> y (C, P, 3) = (s * x) @ R + T."""
    return (s[:, None] * x[None]) @ R + T[:, None]


def chamfer_loss(y: torch.Tensor, g: torch.Tensor) -> torch.Tensor:
    """(C, P, 3), (Q, 3) -> (C,) mean squared distance pred->gt plus gt->pred."""
    d = ((y[:, :, None, :] - g[None, None]) ** 2).sum(-1)         # (C, P, Q)
    return d.min(2).values.mean(1) + d.min(1).values.mean(1)


def nearest(y: torch.Tensor, g: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """Nearest-neighbour indices (lowest index on ties): a (C, P) into g, b (C, Q) into y's points."""
    d = ((y[:, :, None, :] - g[None, None]) ** 2).sum(-1)
    return d.argmin(2), d.argmin(1)


def chamfer_sums(x, g, R, s, T, a=None, b=None) -> torch.Tensor:
    """(C, 13) = loss, t, A (row-major) for candidates (R, s, T), in the dtype of the inputs.  a, b: nearest-neighbour
    choices to use (default: `nearest` in that dtype)."""
    y = transform(x, R, s, T)
    if a is None:
        a, b = nearest(y, g)
    P, Q = x.shape[0], g.shape[0]
    out = []
    for n in range(y.shape[0]):
        e1 = y[n] - g[a[n]]                      # (P, 3)
        e2 = y[n, b[n]] - g                      # (Q, 3)
        loss = (e1 ** 2).sum() / P + (e2 ** 2).sum() / Q
        t = 2 * e1.sum(0) / P + 2 * e2.sum(0) / Q
        A = 2 * x.T @ e1 / P + 2 * x[b[n]].T @ e2 / Q
        out.append(torch.cat([loss[None], t, A.reshape(9)]))
    return torch.stack(out)


def _normalize(v: torch.Tensor) -> torch.Tensor:
    return v / v.norm(dim=-1, keepdim=True).clamp_min(1e-12)


def rot6d_to_matrix(d6: torch.Tensor) -> torch.Tensor:
    """pytorch3d rotation_6d_to_matrix: (..., 6) -> (..., 3, 3), rows b1, b2, b3."""
    a1, a2 = d6[..., :3], d6[..., 3:]
    b1 = _normalize(a1)
    b2 = _normalize(a2 - (b1 * a2).sum(-1, keepdim=True) * b1)
    return torch.stack((b1, b2, torch.cross(b1, b2, dim=-1)), dim=-2)


def _normalize_backward(v: torch.Tensor, g: torch.Tensor) -> torch.Tensor:
    n = v.norm()
    if n > 1e-12:
        b = v / n
        return (g - b * (b @ g)) / n
    return g / 1e-12


def rot6d_backward(d6: torch.Tensor, gm: torch.Tensor) -> torch.Tensor:
    """Closed-form dL/d(d6) (6,) from dL/dM (3, 3) for one 6D vector, in fp64."""
    d6, gm = d6.double(), gm.double()
    a1, a2 = d6[:3], d6[3:]
    b1 = a1 / a1.norm().clamp_min(1e-12)
    u = a2 - (b1 @ a2) * b1
    b2 = u / u.norm().clamp_min(1e-12)
    gb1 = gm[0] + torch.linalg.cross(b2, gm[2])
    gb2 = gm[1] + torch.linalg.cross(gm[2], b1)
    gu = _normalize_backward(u, gb2)
    ga2 = gu - b1 * (b1 @ gu)
    gb1 = gb1 - ((b1 @ a2) * gu + a2 * (b1 @ gu))
    return torch.cat([_normalize_backward(a1, gb1), ga2])


def param_grads(sums: torch.Tensor, rot_init: torch.Tensor, R: torch.Tensor, params: torch.Tensor) -> torch.Tensor:
    """(C, 13) sums, (C, 3, 3) R_init, (C, 3, 3) R, (C, 12) params -> (C, 12) fp64 gradient of loss.mean() over the C
    candidates with respect to (T, d6, s)."""
    C = sums.shape[0]
    sums, R, params, rot_init = sums.double() / C, R.double(), params.double(), rot_init.double()
    out = []
    for n in range(C):
        t, A, s = sums[n, 1:4], sums[n, 4:].reshape(3, 3), params[n, 9:]
        gR = s[:, None] * A
        gs = (R[n] * A).sum(1)
        gd6 = rot6d_backward(params[n, 3:9], rot_init[n].T @ gR)
        out.append(torch.cat([t, gd6, gs]))
    return torch.stack(out)


def adam_step(params, m, v, grad, step: int, lr: float):
    """torch.optim.Adam (betas 0.9 / 0.999, eps 1e-8) on fp32 tensors -> new (params, m, v).  m and v in the order of
    torch's CPU path (v = fl(0.999 v) + fl(fl(0.001 g) g)); torch's CUDA path computes v = fma(0.001, fl(g g), fl(0.999 v)),
    and the params update rounds differently on both, so this is an approximation to a few ulps (DESIGN §12)."""
    grad = grad.float()
    m = torch.lerp(m, grad, 1 - 0.9)
    v = v * 0.999 + (1 - 0.999) * grad * grad
    step_size = lr / (1 - 0.9 ** step)
    denom = v.sqrt() / ((1 - 0.999 ** step) ** 0.5) + 1e-8
    return params - step_size * (m / denom), m, v


def best_update(losses: torch.Tensor, best: torch.Tensor, R_pre: torch.Tensor, params_post: torch.Tensor) -> torch.Tensor:
    """icp.py:99-106 for one frame: best (16,) = loss, R, T, s -> the updated copy."""
    best = best.clone()
    if torch.isnan(losses).any():
        return best
    idx = int(torch.nonzero(losses == losses.min())[0])
    if float(losses[idx]) < float(best[0]):
        best[0] = losses[idx]
        best[1:10] = R_pre[idx].reshape(9)
        best[10:13] = params_post[idx, :3]
        best[13:16] = params_post[idx, 9:]
    return best


def initial_state(C: int):
    """params (C, 12) = T 0, d6 (1, 0, 0, 0, 1, 0), s 1, as icp.py:81-85."""
    params = torch.zeros(C, 12)
    params[:, 3] = 1
    params[:, 7] = 1
    params[:, 9:] = 1
    return params
