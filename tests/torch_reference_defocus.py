"""The dense float64 evaluator of ``torch_reference_motion_blur.dense_render_blur`` with depth of field -- what
``CameraInfo.defocus`` (``gsb200_forward_defocus`` / ``gsb200_backward_defocus``) renders and differentiates (test helper).

Definition in ``include/gsb200.h``: with z the rendered depth (detached) and M = K[:2,:2] D at the detached point,
beta = a^2 (rho - 1/z)^2 / 16 and B_d = beta M M^T is added to the motion blur's B = d d^T / 12; the conic, c_b and the radius
come from Sigma_d + B as for the motion blur.  ``aux`` has ``dense_render_blur``'s fields plus ``blur_px`` = a f |rho - 1/z|,
the disk's diameter in pixels along x.  The image is differentiable in xyz, the features, the exposure motion and (a, rho).
"""
import torch

from torch_reference import quat_to_rot, sh_basis
from torch_reference_lens import distortion_jacobian, project, r2_bound
from torch_reference_pose import camera_from_pose
from torch_reference_rolling_shutter import moved, row_time


def dense_render_defocus(xyz, feats, invalid_mask, object_id, K, q_pc, t_pc, H, W, model, k, motion, blur, defocus, near=0.8,
                         far=1000.0, depth_scale=100.0):
    """``dense_render_blur`` with the thin lens ``defocus`` = (a, rho) (2,).  Differentiable w.r.t. xyz, feats, blur and
    defocus (the row time, and with it ``motion``, is detached here)."""
    dt = torch.float64
    xyz, feats, K = xyz.to(dt), feats.to(dt), K.to(dt)
    m = motion.to(dt) if isinstance(motion, torch.Tensor) else torch.tensor(motion, dtype=dt)
    mb = blur.to(dt) if isinstance(blur, torch.Tensor) else torch.tensor(blur, dtype=dt)
    df = defocus.to(dt) if isinstance(defocus, torch.Tensor) else torch.tensor(defocus, dtype=dt)
    Rc_o, tc_o = camera_from_pose(q_pc.to(dt), t_pc.to(dt))
    oid = object_id.long()
    Rc, tc = Rc_o[oid], tc_o[oid]
    pc0 = (Rc @ xyz[..., None])[..., 0] + tc
    tau = row_time(pc0, K, H, model, k, m)
    pc, Rd = moved(pc0, tau, m)
    z = pc[:, 2]
    uv = project(pc, K, model, k)
    xn, yn = pc[:, 0].detach() / z.detach(), pc[:, 1].detach() / z.detach()
    valid = (xn * xn + yn * yn) <= r2_bound(model, k)
    inside = (invalid_mask.to(torch.bool) == 0) & valid & (z > near) & (z < far) & (uv[:, 0] >= -48) & \
        (uv[:, 0] < W + 48) & (uv[:, 1] >= -48) & (uv[:, 1] < H + 48)
    ids = torch.nonzero(inside.detach()).reshape(-1)
    tau_all = torch.where(inside.detach(), tau, torch.zeros_like(tau))
    pc, uv, z, Rc, tc, Rd = pc[ids], uv[ids], z[ids], Rc[ids], tc[ids], Rd[ids]
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
    U = J @ Rd @ Rc
    cov = U @ Sigma @ U.transpose(-1, -2)
    a0, b0, c0, d0 = cov[:, 0, 0], cov[:, 0, 1], cov[:, 1, 0], cov[:, 1, 1]
    det0 = a0 * d0 - b0 * c0
    a1, d1 = a0 + 0.3, d0 + 0.3
    det1 = a1 * d1 - b0 * c0
    rescale = torch.sqrt(torch.clamp(det0 / det1, min=0.0)).detach()
    # the blur: d = Jp (v + w x pc) with the full position Jacobian at the detached point, B = d d^T / 12
    Jp = K[:2, :2] @ D @ P
    vel = mb[:3][None, :] + torch.cross(mb[3:].expand_as(pcd), pcd, dim=-1)
    d = (Jp @ vel[..., None])[..., 0]
    B = d[:, :, None] * d[:, None, :] / 12.0
    # the defocus: beta = a^2 (rho - 1/z)^2 / 16 at the detached depth, B_d = beta M M^T with M = K[:2,:2] D
    Mk = K[:2, :2] @ D
    e = df[1] - 1.0 / pcd[:, 2]
    beta = df[0] ** 2 * e ** 2 / 16.0
    B = B + beta[:, None, None] * (Mk @ Mk.transpose(-1, -2))
    a2, b2, c2, d2 = a1 + B[:, 0, 0], b0 + B[:, 0, 1], c0 + B[:, 1, 0], d1 + B[:, 1, 1]
    det2 = a2 * d2 - b2 * c2
    comp = torch.sqrt(det1 / det2)  # c_b, differentiable
    ca, cb, cc = d2 / det2, -b2 / det2, a2 / det2
    opacity = torch.sigmoid(logit)
    cam_centre = -(Rc.transpose(-1, -2) @ tc[..., None])[..., 0]
    basis = sh_basis((xyz[ids] - cam_centre).detach())
    color = torch.sigmoid((f[:, 8:56].reshape(M, 3, 16) * basis[:, None, :]).sum(-1))
    ra, rb, rc, rd = a0 + B[:, 0, 0], b0 + B[:, 0, 1], c0 + B[:, 1, 0], d0 + B[:, 1, 1]  # Sigma' + B
    lam = (ra + rd + torch.sqrt((ra - rd) ** 2 + 4 * rb * rc)) / 2
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
    for mm in order.tolist():
        member = (ptu >= min_tu[mm]) & (ptu < max_tu[mm]) & (ptv >= min_tv[mm]) & (ptv < max_tv[mm])
        if not bool(member.any()):
            continue
        dx, dy = px - uv[mm, 0], py - uv[mm, 1]
        alpha = torch.exp(-0.5 * (dx * dx * ca[mm] + dy * dy * cc[mm]) - dx * dy * cb[mm]) * rescale[mm] * comp[mm] * opacity[mm]
        active = member & ~stopped & (alpha.detach() >= 1.0 / 255.0)
        alpha_c = alpha + (torch.clamp(alpha, max=0.99) - alpha).detach()
        nT = T * (1 - alpha_c)
        stop_now = active & (nT.detach() < 1e-4)
        stopped = stopped | stop_now
        blend = active & ~stop_now
        w = alpha_c * T
        C = C + torch.where(blend[..., None], color[mm][None, None, :] * w[..., None], torch.zeros_like(C))
        cnt = cnt + blend.to(torch.int32)
        T = torch.where(blend, nT, T)
    aux = dict(ids=ids, uv=uv, pc=pc, conic=torch.stack([ca, cb, cc, rescale], -1), opacity=opacity * comp, color=color,
               radius=radius, acc_alpha=1 - T, count=cnt, tau=tau_all, comp=comp, streak=torch.sqrt((d * d).sum(-1)),
               blur_px=(torch.abs(df[0] * e) * K[0, 0]).detach())
    return C, aux
