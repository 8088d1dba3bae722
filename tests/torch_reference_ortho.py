"""The dense float64 evaluator of an orthographic view -- what ``LensDistortion("orthographic", ())`` (``gsb200_forward_ortho``
/ ``gsb200_backward_ortho``) renders and differentiates (test helper).

The model is the one of ``include/gsb200.h``: pc = W xyz + t (the pose as ``torch_reference_pose.camera_from_pose`` maps it),
u = K00 x + K01 y + K02, v = K10 x + K11 y + K12; J = K[:2,:2] [I 0], not detached (it does not depend on pc); in view when
near < z < far and (u, v) lies inside the image plus three boundary tiles; depth z; SH view direction row 2 of W (detached).
With ``filter3d`` the 3D smoothing filter of ``mip_filter``: scales sqrt(exp(s)^2 + sigma^2) and the opacity compensation
sqrt(prod exp(s)^2 / (exp(s)^2 + sigma^2)), differentiable in s.  Everything else -- the conventions (the 0.3 low-pass'
``rescale`` detached, the 0.99 clamp straight-through), the pinhole's tile rectangle, depth order, 1/255 cut and 1e-4 early
stop -- is ``torch_reference.dense_render``'s.  Differentiable in xyz, feats, q_pc, t_pc, K and the extra features."""
import torch

from torch_reference import quat_to_rot, sh_basis
from torch_reference_pose import camera_from_pose


def dense_render_ortho(xyz, feats, invalid_mask, object_id, K, q_pc, t_pc, H, W, near=0.8, far=1000.0, extra_features=None,
                       filter3d=None):
    """Returns (image (H,W,3), depth (H,W), acc_alpha (H,W), feature map (H,W,C) or None, aux), all f64."""
    dt = torch.float64
    xyz, feats, K = xyz.to(dt), feats.to(dt), K.to(dt)
    Rc_o, tc_o = camera_from_pose(q_pc.to(dt), t_pc.to(dt))
    oid = object_id.long()
    Rc, tc = Rc_o[oid], tc_o[oid]
    pc = (Rc @ xyz[..., None])[..., 0] + tc
    z = pc[:, 2]
    uv = pc[:, :2] @ K[:2, :2].T + K[:2, 2]
    inside = (invalid_mask.to(torch.bool) == 0) & (z > near) & (z < far) & (uv[:, 0] >= -48) & (uv[:, 0] < W + 48) & \
        (uv[:, 1] >= -48) & (uv[:, 1] < H + 48)
    ids = torch.nonzero(inside.detach()).reshape(-1)
    pc, uv, z, Rc = pc[ids], uv[ids], z[ids], Rc[ids]
    f = feats[ids]
    M = ids.shape[0]
    q, s, logit = f[:, 0:4], f[:, 4:7], f[:, 7]
    J = torch.cat([K[:2, :2], torch.zeros((2, 1), dtype=dt)], 1).expand(M, 2, 3)
    R = quat_to_rot(q)
    e = torch.exp(2 * s)
    comp = torch.ones(M, dtype=dt)
    if filter3d is not None:
        s2 = torch.clamp(filter3d.to(dt)[ids], min=0.0) ** 2
        eh = e + s2[:, None]
        comp = torch.sqrt(torch.prod(e / eh, -1))
        e = eh
    Sigma = R @ torch.diag_embed(e) @ R.transpose(-1, -2)
    U = J @ Rc
    cov = U @ Sigma @ U.transpose(-1, -2)
    a0, b0, c0, d0 = cov[:, 0, 0], cov[:, 0, 1], cov[:, 1, 0], cov[:, 1, 1]
    det0 = a0 * d0 - b0 * c0
    a1, d1 = a0 + 0.3, d0 + 0.3
    det1 = a1 * d1 - b0 * c0
    rescale = torch.sqrt(torch.clamp(det0 / det1, min=0.0)).detach() * comp
    ca, cb, cc = d1 / det1, -b0 / det1, a1 / det1
    opacity = torch.sigmoid(logit)
    basis = sh_basis(Rc[:, 2, :].detach())
    color = torch.sigmoid((f[:, 8:56].reshape(M, 3, 16) * basis[:, None, :]).sum(-1))
    lam = (a0 + d0 + torch.sqrt((a0 - d0) ** 2 + 4 * b0 * c0)) / 2
    radius = (3.0 * torch.sqrt(lam)).detach().to(torch.float32)
    uvf = uv.detach().to(torch.float32)
    r = torch.clamp(radius, min=1.0)
    th, tw = H // 16, W // 16
    min_tu = torch.clamp(torch.floor(torch.clamp(uvf[:, 0] - r, min=0.0) / 16).to(torch.int64), max=tw)
    max_tu = torch.clamp(torch.maximum(torch.floor((uvf[:, 0] + r) / 16).to(torch.int64) + 1, min_tu + 1), max=tw)
    min_tv = torch.clamp(torch.floor(torch.clamp(uvf[:, 1] - r, min=0.0) / 16).to(torch.int64), max=th)
    max_tv = torch.clamp(torch.maximum(torch.floor((uvf[:, 1] + r) / 16).to(torch.int64) + 1, min_tv + 1), max=th)
    depth_key = (z.detach().to(torch.float32) * torch.tensor(100.0, dtype=torch.float32)).to(torch.int32)
    order = torch.argsort(depth_key.to(torch.int64) * (M + 1) + torch.arange(M), stable=True)
    ys, xs = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    px, py = xs.to(dt) + 0.5, ys.to(dt) + 0.5
    ptu, ptv = xs // 16, ys // 16
    T = torch.ones((H, W), dtype=dt)
    C = torch.zeros((H, W, 3), dtype=dt)
    Dn = torch.zeros((H, W), dtype=dt)
    ef = None if extra_features is None else extra_features.to(dt)[ids]
    F = None if ef is None else torch.zeros((H, W, ef.shape[1]), dtype=dt)
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
        w = torch.where(blend, alpha_c * T, torch.zeros_like(T))
        C = C + color[m][None, None, :] * w[..., None]
        Dn = Dn + z[m] * w
        if F is not None:
            F = F + ef[m][None, None, :] * w[..., None]
        T = torch.where(blend, nT, T)
    S = 1 - T
    depth = Dn / torch.clamp(S, min=1e-6)
    aux = dict(ids=ids, uv=uv, pc=pc, depth=z, conic=torch.stack([ca, cb, cc, rescale], -1), opacity=opacity, color=color,
               radius=radius, min_tu=min_tu, max_tu=max_tu, min_tv=min_tv, max_tv=max_tv)
    return C, depth, S, F, aux
