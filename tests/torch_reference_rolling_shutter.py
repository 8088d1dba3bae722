"""The dense float64 evaluator of ``torch_reference_lens.dense_render_lens`` through a rolling shutter -- what
``CameraInfo.rolling_shutter`` (``gsb200_forward_rolling_shutter`` / ``gsb200_backward_rolling_shutter``) renders and
differentiates (test helper).

Definition in ``include/gsb200.h``: with pc0 = W xyz + tw, the row time tau is the GSB_RS_ITERATIONS = 3 fixed-point steps
tau <- clamp(v_pix(pc(tau)) / H - 1/2, -1/2, 1/2) from 0 (detached), the point is rendered at pc(tau) = Rd(tau) pc0 + tau v
with Rd(tau) = exp(tau [w]x), and Sigma' uses J Rd W.  The SH view direction keeps the mid-readout camera centre.  Everything
else is ``dense_render_lens``'s, and ``aux`` has its fields (plus ``tau``, the row time of every scene row), so
``torch_reference_depth.differentiable_depth`` and ``torch_reference_features.feature_map`` work on it unchanged.  The image is
differentiable in xyz, the features and the motion m = (v, w)."""
import torch

from torch_reference import quat_to_rot, sh_basis
from torch_reference_lens import distortion_jacobian, project, r2_bound
from torch_reference_pose import camera_from_pose

ITERATIONS = 3


def hat(p):
    """(M,3) -> (M,3,3) cross-product matrices."""
    z = torch.zeros_like(p[:, 0])
    return torch.stack([torch.stack([z, -p[:, 2], p[:, 1]], -1), torch.stack([p[:, 2], z, -p[:, 0]], -1),
                        torch.stack([-p[:, 1], p[:, 0], z], -1)], -2)


def rodrigues(p):
    """exp([p]x) per row in float64, differentiable (also at p = 0)."""
    t2 = (p * p).sum(-1)
    small = t2 < 1e-8
    ts = torch.where(small, torch.ones_like(t2), t2)
    th = torch.sqrt(ts)
    A = torch.where(small, 1 - t2 / 6, torch.sin(th) / th)
    B = torch.where(small, 0.5 - t2 / 24, (1 - torch.cos(th)) / ts)
    P = hat(p)
    eye = torch.eye(3, dtype=p.dtype).expand(p.shape[0], 3, 3)
    return eye + A[:, None, None] * P + B[:, None, None] * (P @ P)


def moved(pc0, tau, m):
    """pc(tau) = Rd(tau) pc0 + tau v and Rd(tau), per row."""
    R = rodrigues(tau[:, None] * m[3:][None, :])
    return (R @ pc0[..., None])[..., 0] + tau[:, None] * m[:3][None, :], R


def row_time(pc0, K, H, model, k, m):
    """The detached fixed-point row time of every row."""
    with torch.no_grad():
        pc0, m = pc0.detach(), m.detach()
        tau = torch.zeros_like(pc0[:, 0])
        for _ in range(ITERATIONS):
            pt, _ = moved(pc0, tau, m)
            r = project(pt, K, model, k)[:, 1] / H - 0.5
            tau = torch.clamp(torch.nan_to_num(r, nan=-0.5), -0.5, 0.5)
    return tau


def dense_render_rs(xyz, feats, invalid_mask, object_id, K, q_pc, t_pc, H, W, model, k, motion, near=0.8, far=1000.0,
                    depth_scale=100.0):
    """Multi-object scene through the lens (model, k; "pinhole": none) and the rolling shutter of ``motion`` (6,).  Returns the
    image (H,W,3) f64 and the intermediates; differentiable w.r.t. xyz, feats and motion."""
    dt = torch.float64
    xyz, feats, K = xyz.to(dt), feats.to(dt), K.to(dt)
    m = motion.to(dt) if isinstance(motion, torch.Tensor) else torch.tensor(motion, dtype=dt)
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
    for mm in order.tolist():
        member = (ptu >= min_tu[mm]) & (ptu < max_tu[mm]) & (ptv >= min_tv[mm]) & (ptv < max_tv[mm])
        if not bool(member.any()):
            continue
        dx, dy = px - uv[mm, 0], py - uv[mm, 1]
        alpha = torch.exp(-0.5 * (dx * dx * ca[mm] + dy * dy * cc[mm]) - dx * dy * cb[mm]) * rescale[mm] * opacity[mm]
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
    aux = dict(ids=ids, uv=uv, pc=pc, conic=torch.stack([ca, cb, cc, rescale], -1), opacity=opacity, color=color,
               radius=radius, acc_alpha=1 - T, count=cnt, tau=tau_all)
    return C, aux
