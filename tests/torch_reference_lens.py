"""The dense float64 evaluator of ``torch_reference_pose.dense_render_objects`` through a distorting lens -- what
``CameraInfo.distortion`` (``gsb200_forward_lens`` / ``gsb200_backward_lens``) renders and differentiates (test helper).

The lens acts between the camera-frame point and K (definition in ``include/gsb200.h``): uv = K[:2,:2] (xd, yd) + K[:2,2],
and J = diag(fx, fy) D P inside Sigma' with D = d(xd, yd)/d(xn, yn) taken by autograd at the detached point.  A point with
r^2 > r_max^2 is outside the frustum.  Everything else -- the conventions (J, the SH view direction and ``rescale`` detached,
the 0.99 clamp straight-through), tile membership, depth order, 1/255 cut and 1e-4 early stop -- is ``dense_render``'s, and
``aux`` has its fields, so ``torch_reference_depth.differentiable_depth`` and ``torch_reference_features.feature_map`` work
on it unchanged."""
import math

import numpy as np
import torch

from torch_reference import quat_to_rot, sh_basis
from torch_reference_pose import camera_from_pose

MODELS = {"pinhole": 0, "opencv": 1, "fisheye": 2}


def distort(xn, yn, model, k):
    """(xn, yn) -> (xd, yd) in float64, differentiable, finite on the optical axis."""
    if model == "pinhole":
        return xn, yn
    r2 = xn * xn + yn * yn
    if model == "opencv":
        k1, k2, p1, p2, k3 = (float(v) for v in k)
        rad = 1 + k1 * r2 + k2 * r2 ** 2 + k3 * r2 ** 3
        return (xn * rad + 2 * p1 * xn * yn + p2 * (r2 + 2 * xn * xn),
                yn * rad + p1 * (r2 + 2 * yn * yn) + 2 * p2 * xn * yn)
    assert model == "fisheye"
    k1, k2, k3, k4 = (float(v) for v in k[:4])
    small = r2 < 1e-12
    r = torch.sqrt(torch.where(small, torch.ones_like(r2), r2))
    theta = torch.atan(r)
    t2 = theta * theta
    td_over_r = theta * (1 + k1 * t2 + k2 * t2 ** 2 + k3 * t2 ** 3 + k4 * t2 ** 4) / r
    # theta_d / r = 1 + (k1 - 1/3) r^2 + O(r^4) on the axis
    s = torch.where(small, 1 + (k1 - 1.0 / 3.0) * r2, td_over_r)
    return s * xn, s * yn


def project(pc, K, model, k):
    """(M,3) camera-frame points -> (M,2) pixel positions through the lens, float64, differentiable in pc."""
    z = pc[:, 2]
    xd, yd = distort(pc[:, 0] / z, pc[:, 1] / z, model, k)
    return torch.stack([K[0, 0] * xd + K[0, 1] * yd + K[0, 2], K[1, 0] * xd + K[1, 1] * yd + K[1, 2]], -1)


def distortion_jacobian(xn, yn, model, k):
    """D = d(xd, yd)/d(xn, yn) per point by autograd, (M,2,2), detached."""
    xn = xn.detach().clone().requires_grad_(True)
    yn = yn.detach().clone().requires_grad_(True)
    with torch.enable_grad():
        xd, yd = distort(xn, yn, model, k)
        gx = torch.autograd.grad(xd.sum(), (xn, yn), retain_graph=True, allow_unused=True)
        gy = torch.autograd.grad(yd.sum(), (xn, yn), allow_unused=True)
    z = torch.zeros_like(xn)
    fix = lambda g: z if g is None else g  # noqa: E731
    return torch.stack([torch.stack([fix(gx[0]), fix(gx[1])], -1), torch.stack([fix(gy[0]), fix(gy[1])], -1)], -2).detach()


def r2_bound(model, k):
    """r_max^2 of the definition in float64 from numpy's polynomial roots (inf when the map never folds back)."""
    if model == "opencv":
        c = [1.0, 3.0 * k[0], 5.0 * k[1], 7.0 * k[4]]
        roots = np.roots(c[::-1]) if any(c[1:]) else []
        pos = [x.real for x in np.atleast_1d(roots) if abs(x.imag) < 1e-12 and x.real > 0]
        return min(pos) if pos else math.inf
    if model == "fisheye":
        c = [1.0, 3.0 * k[0], 5.0 * k[1], 7.0 * k[2], 9.0 * k[3]]
        roots = np.roots(c[::-1]) if any(c[1:]) else []
        pos = [x.real for x in np.atleast_1d(roots) if abs(x.imag) < 1e-12 and 0 < x.real < (math.pi / 2) ** 2]
        if not pos:
            return math.inf
        return math.tan(math.sqrt(min(pos))) ** 2
    return math.inf


def dense_render_lens(xyz, feats, invalid_mask, object_id, K, q_pc, t_pc, H, W, model, k, near=0.8, far=1000.0,
                      depth_scale=100.0):
    """Multi-object scene through the lens (model, k).  Returns the image (H,W,3) f64 and the intermediates of
    ``dense_render``; differentiable w.r.t. xyz, feats, q_pc and t_pc."""
    dt = torch.float64
    xyz, feats, K = xyz.to(dt), feats.to(dt), K.to(dt)
    Rc_o, tc_o = camera_from_pose(q_pc.to(dt), t_pc.to(dt))
    oid = object_id.long()
    Rc, tc = Rc_o[oid], tc_o[oid]
    pc = (Rc @ xyz[..., None])[..., 0] + tc
    z = pc[:, 2]
    uv = project(pc, K, model, k)
    xn, yn = pc[:, 0].detach() / z.detach(), pc[:, 1].detach() / z.detach()
    valid = (xn * xn + yn * yn) <= r2_bound(model, k)
    inside = (invalid_mask.to(torch.bool) == 0) & valid & (z > near) & (z < far) & (uv[:, 0] >= -48) & \
        (uv[:, 0] < W + 48) & (uv[:, 1] >= -48) & (uv[:, 1] < H + 48)
    ids = torch.nonzero(inside.detach()).reshape(-1)
    pc, uv, z, Rc, tc = pc[ids], uv[ids], z[ids], Rc[ids], tc[ids]
    f = feats[ids]
    M = ids.shape[0]
    q, s, logit = f[:, 0:4], f[:, 4:7], f[:, 7]
    pcd = pc.detach()
    D = distortion_jacobian(pcd[:, 0] / pcd[:, 2], pcd[:, 1] / pcd[:, 2], model, k)
    zeros = torch.zeros_like(pcd[:, 0])
    P = torch.stack([torch.stack([1 / pcd[:, 2], zeros, -pcd[:, 0] / pcd[:, 2] ** 2], -1),
                     torch.stack([zeros, 1 / pcd[:, 2], -pcd[:, 1] / pcd[:, 2] ** 2], -1)], -2)
    J = torch.diag(torch.stack([K[0, 0], K[1, 1]])).to(dt) @ D @ P
    R = quat_to_rot(q)
    Sigma = R @ torch.diag_embed(torch.exp(2 * s)) @ R.transpose(-1, -2)
    U = J @ Rc
    cov = U @ Sigma @ U.transpose(-1, -2)
    a0, b0, c0, d0 = cov[:, 0, 0], cov[:, 0, 1], cov[:, 1, 0], cov[:, 1, 1]
    det0 = a0 * d0 - b0 * c0
    a1, d1 = a0 + 0.3, d0 + 0.3
    det1 = a1 * d1 - b0 * c0
    rescale = torch.sqrt(torch.clamp(det0 / det1, min=0.0)).detach()
    ca, cb, cc = d1 / det1, -b0 / det1, a1 / det1
    opacity = torch.sigmoid(logit)
    cam_centre = -(Rc.transpose(-1, -2) @ tc[..., None])[..., 0]
    basis = sh_basis((xyz[ids] - cam_centre).detach())
    color = torch.sigmoid((f[:, 8:56].reshape(M, 3, 16) * basis[:, None, :]).sum(-1))
    lam = (a0 + d0 + torch.sqrt((a0 - d0) ** 2 + 4 * b0 * c0)) / 2
    radius = (3.0 * torch.sqrt(lam)).detach().to(torch.float32)
    uvf = uv.detach().to(torch.float32)
    r = torch.clamp(radius, min=1.0)
    tw, th = W // 16, H // 16
    min_tu = torch.clamp(torch.floor(torch.clamp(uvf[:, 0] - r, min=0.0) / 16).to(torch.int64), max=tw)
    max_tu = torch.clamp(torch.maximum(torch.floor((uvf[:, 0] + r) / 16).to(torch.int64) + 1, min_tu + 1), max=tw)
    min_tv = torch.clamp(torch.floor(torch.clamp(uvf[:, 1] - r, min=0.0) / 16).to(torch.int64), max=th)
    max_tv = torch.clamp(torch.maximum(torch.floor((uvf[:, 1] + r) / 16).to(torch.int64) + 1, min_tv + 1), max=th)
    depth_key = (z.detach().to(torch.float32) * torch.tensor(depth_scale, dtype=torch.float32)).to(torch.int32)
    order = torch.argsort(depth_key.to(torch.int64) * (M + 1) + torch.arange(M), stable=True)
    ys, xs = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    px, py = xs.to(dt) + 0.5, ys.to(dt) + 0.5
    ptu, ptv = xs // 16, ys // 16
    T = torch.ones((H, W), dtype=dt)
    C = torch.zeros((H, W, 3), dtype=dt)
    cnt = torch.zeros((H, W), dtype=torch.int32)
    stopped = torch.zeros((H, W), dtype=torch.bool)
    for m in order.tolist():
        member = (ptu >= min_tu[m]) & (ptu < max_tu[m]) & (ptv >= min_tv[m]) & (ptv < max_tv[m])
        if not bool(member.any()):
            continue
        dx, dy = px - uv[m, 0], py - uv[m, 1]
        alpha = torch.exp(-0.5 * (dx * dx * ca[m] + dy * dy * cc[m]) - dx * dy * cb[m]) * rescale[m] * opacity[m]
        active = member & ~stopped & (alpha.detach() >= 1.0 / 255.0)
        alpha_c = alpha + (torch.clamp(alpha, max=0.99) - alpha).detach()
        nT = T * (1 - alpha_c)
        stop_now = active & (nT.detach() < 1e-4)
        stopped = stopped | stop_now
        blend = active & ~stop_now
        w = alpha_c * T
        C = C + torch.where(blend[..., None], color[m][None, None, :] * w[..., None], torch.zeros_like(C))
        cnt = cnt + blend.to(torch.int32)
        T = torch.where(blend, nT, T)
    aux = dict(ids=ids, uv=uv, pc=pc, conic=torch.stack([ca, cb, cc, rescale], -1), opacity=opacity, color=color,
               radius=radius, acc_alpha=1 - T, count=cnt)
    return C, aux
