"""The dense float64 evaluator of an equirectangular panorama -- what ``LensDistortion("equirectangular", ())``
(``gsb200_forward_equirect`` / ``gsb200_backward_equirect``) renders and differentiates (test helper).

The model is the one of ``include/gsb200.h``: rho = |(x, z)|, r = |pc|, u = fx atan2(x, z) + cx reduced into [0, W),
v = fy atan2(y, rho) + cy; J = diag(fx, fy) [z/rho^2 0 -x/rho^2; -xy/(r^2 rho) rho/r^2 -zy/(r^2 rho)] at the detached point
inside Sigma'; in view when near < r < far and rho > 1e-3 r; depth r.  A pixel sees a splat when its tile column is one of
the splat's columns modulo W/16 and its tile row one of its rows, at the copy of u nearest the tile's centre column.
Everything else -- the conventions (J, the SH view direction and ``rescale`` detached, the 0.99 clamp straight-through), depth
order, 1/255 cut and 1e-4 early stop -- is ``torch_reference.dense_render``'s."""
import math

import numpy as np
import torch

from torch_reference import quat_to_rot, sh_basis
from torch_reference_pose import camera_from_pose

POLE_EPSILON = 1e-3


def project(pc, K, W):
    """(u, v) of camera-frame points (M,3) f64, u reduced into [0, W); differentiable."""
    x, y, z = pc[:, 0], pc[:, 1], pc[:, 2]
    rho = torch.sqrt(x * x + z * z)
    u = K[0, 0] * torch.atan2(x, z) + K[0, 2]
    u = u - W * torch.floor(u.detach() / W)
    v = K[1, 1] * torch.atan2(y, rho) + K[1, 2]
    return torch.stack([u, v], -1)


def jacobian(pcd, K):
    """J (M,2,3) at detached points."""
    x, y, z = pcd[:, 0], pcd[:, 1], pcd[:, 2]
    rho2 = x * x + z * z
    rho = torch.sqrt(rho2)
    r2 = rho2 + y * y
    zeros = torch.zeros_like(x)
    J = torch.stack([torch.stack([K[0, 0] * z / rho2, zeros, -K[0, 0] * x / rho2], -1),
                     torch.stack([-K[1, 1] * x * y / (r2 * rho), K[1, 1] * rho / r2, -K[1, 1] * z * y / (r2 * rho)], -1)], -2)
    return J


def columns(u, radius, W):
    """The footprint's unwrapped tile columns [a, b) (equirect_columns of csrc/preprocess.cu), f32 inputs."""
    tw = W // 16
    r = torch.clamp(radius, min=1.0)
    fa = torch.floor((u - r) / 16)
    fb = torch.floor((u + r) / 16) + 1
    wide = ~(fb - fa <= tw)
    a_wide = torch.ceil((u - 0.5 * W - 8.0) / 16)
    a = torch.where(wide, a_wide, fa)
    b = torch.where(wide, a_wide + tw, fb)
    return a.to(torch.int64), b.to(torch.int64)


def dense_render_equirect(xyz, feats, invalid_mask, object_id, K, q_pc, t_pc, H, W, near=0.8, far=1000.0,
                          extra_features=None):
    """Returns (image (H,W,3), depth (H,W), acc_alpha (H,W), feature map (H,W,C) or None, aux), all f64 and differentiable
    w.r.t. xyz, feats and ``extra_features``."""
    dt = torch.float64
    xyz, feats, K = xyz.to(dt), feats.to(dt), K.to(dt)
    Rc_o, tc_o = camera_from_pose(q_pc.to(dt), t_pc.to(dt))
    oid = object_id.long()
    Rc, tc = Rc_o[oid], tc_o[oid]
    pc = (Rc @ xyz[..., None])[..., 0] + tc
    rd = pc.norm(dim=-1)
    rho = torch.sqrt(pc[:, 0] ** 2 + pc[:, 2] ** 2)
    uv = project(pc, K, W)
    inside = (invalid_mask.to(torch.bool) == 0) & (rd > near) & (rd < far) & (rho > POLE_EPSILON * rd) & \
        (uv[:, 1] >= -48) & (uv[:, 1] < H + 48)
    ids = torch.nonzero(inside.detach()).reshape(-1)
    pc, uv, rd, Rc, tc = pc[ids], uv[ids], rd[ids], Rc[ids], tc[ids]
    f = feats[ids]
    M = ids.shape[0]
    q, s, logit = f[:, 0:4], f[:, 4:7], f[:, 7]
    J = jacobian(pc.detach(), K)
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
    min_tu, max_tu = columns(uvf[:, 0], radius, W)
    r = torch.clamp(radius, min=1.0)
    th, tw = H // 16, W // 16
    min_tv = torch.clamp(torch.floor(torch.clamp(uvf[:, 1] - r, min=0.0) / 16).to(torch.int64), max=th)
    max_tv = torch.clamp(torch.maximum(torch.floor((uvf[:, 1] + r) / 16).to(torch.int64) + 1, min_tv + 1), max=th)
    depth_key = (rd.detach().to(torch.float32) * torch.tensor(100.0, dtype=torch.float32)).to(torch.int32)
    order = torch.argsort(depth_key.to(torch.int64) * (M + 1) + torch.arange(M), stable=True)
    ys, xs = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    px, py = xs.to(dt) + 0.5, ys.to(dt) + 0.5
    ptu, ptv = xs // 16, ys // 16
    tile_centre = (ptu * 16 + 8).to(dt)
    T = torch.ones((H, W), dtype=dt)
    C = torch.zeros((H, W, 3), dtype=dt)
    Dn = torch.zeros((H, W), dtype=dt)
    ef = None if extra_features is None else extra_features.to(dt)[ids]
    F = None if ef is None else torch.zeros((H, W, ef.shape[1]), dtype=dt)
    stopped = torch.zeros((H, W), dtype=torch.bool)
    for m in order.tolist():
        span = int(max_tu[m] - min_tu[m])
        col_member = ((ptu - min_tu[m]) % tw) < span
        member = col_member & (ptv >= min_tv[m]) & (ptv < max_tv[m])
        if not bool(member.any()):
            continue
        um = uv[m, 0] + W * torch.round((tile_centre - uv[m, 0].detach()) / W)  # round half to even, as rintf
        dx, dy = px - um, py - uv[m, 1]
        alpha = torch.exp(-0.5 * (dx * dx * ca[m] + dy * dy * cc[m]) - dx * dy * cb[m]) * rescale[m] * opacity[m]
        active = member & ~stopped & (alpha.detach() >= 1.0 / 255.0)
        alpha_c = alpha + (torch.clamp(alpha, max=0.99) - alpha).detach()
        nT = T * (1 - alpha_c)
        stop_now = active & (nT.detach() < 1e-4)
        stopped = stopped | stop_now
        blend = active & ~stop_now
        w = torch.where(blend, alpha_c * T, torch.zeros_like(T))
        C = C + color[m][None, None, :] * w[..., None]
        Dn = Dn + rd[m] * w
        if F is not None:
            F = F + ef[m][None, None, :] * w[..., None]
        T = torch.where(blend, nT, T)
    S = 1 - T
    depth = Dn / torch.clamp(S, min=1e-6)
    aux = dict(ids=ids, uv=uv, pc=pc, depth=rd, conic=torch.stack([ca, cb, cc, rescale], -1), opacity=opacity, color=color,
               radius=radius, min_tu=min_tu, max_tu=max_tu, min_tv=min_tv, max_tv=max_tv)
    return C, depth, S, F, aux


def keyed_tiles(aux, W, m):
    """The tile ids the splat m of ``aux`` may key (before the reach filter): columns modulo W/16."""
    tw = W // 16
    out = set()
    for tu in range(int(aux["min_tu"][m]), int(aux["max_tu"][m])):
        for tv in range(int(aux["min_tv"][m]), int(aux["max_tv"][m])):
            out.add(tu % tw + tv * tw)
    return out
