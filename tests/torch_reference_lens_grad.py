"""The dense float64 lens evaluator of ``torch_reference_lens`` with the coefficients as an autograd leaf -- what
``gsb200_backward_lens_grad`` differentiates (test helper).

``distort_k`` / ``project_k`` are ``torch_reference_lens.distort`` / ``project`` with k a float64 tensor.  In the dense
evaluator, D = d(xd, yd)/d(xn, yn) is taken by autograd at the detached point with ``create_graph``, so it stays
differentiable in k but not in the point (the definition in ``include/gsb200.h``); r_max is computed from k's values and not
differentiated.  Everything else is ``dense_render_lens``'s, which ``dense_render_lens_k`` runs with these three pieces
swapped in."""
import contextlib

import torch

import torch_reference_lens as trl


def distort_k(xn, yn, model, k):
    """(xn, yn) -> (xd, yd) in float64, differentiable in the point and in the coefficient tensor k."""
    r2 = xn * xn + yn * yn
    if model == "opencv":
        k1, k2, p1, p2, k3 = k[0], k[1], k[2], k[3], k[4]
        rad = 1 + k1 * r2 + k2 * r2 ** 2 + k3 * r2 ** 3
        return (xn * rad + 2 * p1 * xn * yn + p2 * (r2 + 2 * xn * xn),
                yn * rad + p1 * (r2 + 2 * yn * yn) + 2 * p2 * xn * yn)
    assert model == "fisheye"
    k1, k2, k3, k4 = k[0], k[1], k[2], k[3]
    small = r2 < 1e-12
    r = torch.sqrt(torch.where(small, torch.ones_like(r2), r2))
    theta = torch.atan(r)
    t2 = theta * theta
    td_over_r = theta * (1 + k1 * t2 + k2 * t2 ** 2 + k3 * t2 ** 3 + k4 * t2 ** 4) / r
    s = torch.where(small, 1 + (k1 - 1.0 / 3.0) * r2, td_over_r)
    return s * xn, s * yn


def project_k(pc, K, model, k):
    """(M,3) camera-frame points -> (M,2) pixel positions, float64, differentiable in pc and k."""
    z = pc[:, 2]
    xd, yd = distort_k(pc[:, 0] / z, pc[:, 1] / z, model, k)
    return torch.stack([K[0, 0] * xd + K[0, 1] * yd + K[0, 2], K[1, 0] * xd + K[1, 1] * yd + K[1, 2]], -1)


def distortion_jacobian_k(xn, yn, model, k):
    """D per point, (M,2,2), at the detached point and differentiable in k."""
    xn = xn.detach().clone().requires_grad_(True)
    yn = yn.detach().clone().requires_grad_(True)
    with torch.enable_grad():
        xd, yd = distort_k(xn, yn, model, k)
        gx = torch.autograd.grad(xd.sum(), (xn, yn), create_graph=True)
        gy = torch.autograd.grad(yd.sum(), (xn, yn), create_graph=True)
    return torch.stack([torch.stack([gx[0], gx[1]], -1), torch.stack([gy[0], gy[1]], -1)], -2)


@contextlib.contextmanager
def _coefficients_as_tensor():
    saved = trl.project, trl.distortion_jacobian, trl.r2_bound
    trl.project, trl.distortion_jacobian = project_k, distortion_jacobian_k
    trl.r2_bound = lambda model, k: saved[2](model, k.detach().tolist())
    try:
        yield
    finally:
        trl.project, trl.distortion_jacobian, trl.r2_bound = saved


def dense_render_lens_k(xyz, feats, invalid_mask, object_id, K, q_pc, t_pc, H, W, model, k, **kw):
    """``torch_reference_lens.dense_render_lens`` with k an (n,) float64 tensor (n = 5 for opencv, 4 for fisheye); the image
    and ``aux`` are differentiable in k as well."""
    with _coefficients_as_tensor():
        return trl.dense_render_lens(xyz, feats, invalid_mask, object_id, K, q_pc, t_pc, H, W, model, k, **kw)
