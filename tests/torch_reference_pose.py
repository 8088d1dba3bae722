"""The dense float64 evaluator of ``torch_reference.dense_render`` for a scene of several objects, differentiable in each
object's camera pose (q_pointcloud_camera, t_pointcloud_camera) as well -- what ``differentiable_pose=True`` of the operator
differentiates (test helper).

The pose enters exactly as the library's pose kernel (``csrc/preprocess.cu``) maps it: qi = conj(q_pc) with the rotation
polynomial taken on qi as given, and the translation -R(qi / |qi|) t_pc.  Object o's points are at pc = R(qi_o) xyz + t_o.
Everything else is ``dense_render``: the same conventions (J, the SH view direction and ``rescale`` detached, the 0.99 clamp
straight-through), the same tile-membership mask, depth order, 1/255 cut and 1e-4 early stop.  The returned ``aux`` has
the fields ``dense_render`` returns, so ``torch_reference_depth.differentiable_depth`` and
``torch_reference_features.feature_map`` composite the depth and feature maps on the same graph, and ``aux["acc_alpha"]``
is the differentiable accumulated alpha."""
import torch

from torch_reference import quat_to_rot, sh_basis


def camera_from_pose(q_pc, t_pc):
    """(K,4), (K,3) -> per-object rotation (K,3,3) and translation (K,3) of pc = R xyz + t, as pose_kernel maps them."""
    qi = torch.cat([-q_pc[:, :3], q_pc[:, 3:]], dim=-1)
    qn = qi / qi.norm(dim=-1, keepdim=True)
    return quat_to_rot(qi), -(quat_to_rot(qn) @ t_pc[..., None])[..., 0]


def dense_render_objects(xyz, feats, invalid_mask, object_id, K, q_pc, t_pc, H, W, near=0.8, far=1000.0, depth_scale=100.0):
    """Multi-object scene.  xyz (N,3), feats (N,56) (q assumed unit), object_id (N,), q_pc (K,4), t_pc (K,3).  Returns the
    image (H,W,3) f64 and the intermediates of ``dense_render``; differentiable w.r.t. xyz, feats, q_pc and t_pc."""
    dt = torch.float64
    xyz, feats, K = xyz.to(dt), feats.to(dt), K.to(dt)
    Rc_o, tc_o = camera_from_pose(q_pc.to(dt), t_pc.to(dt))
    oid = object_id.long()
    Rc, tc = Rc_o[oid], tc_o[oid]
    pc = (Rc @ xyz[..., None])[..., 0] + tc
    z = pc[:, 2]
    uv = ((pc @ K.T) / z[:, None])[:, :2]
    inside = (invalid_mask.to(torch.bool) == 0) & (z > near) & (z < far) & (uv[:, 0] >= -48) & \
        (uv[:, 0] < W + 48) & (uv[:, 1] >= -48) & (uv[:, 1] < H + 48)
    ids = torch.nonzero(inside.detach()).reshape(-1)
    pc, uv, z, Rc, tc = pc[ids], uv[ids], z[ids], Rc[ids], tc[ids]
    f = feats[ids]
    M = ids.shape[0]
    q, s, logit = f[:, 0:4], f[:, 4:7], f[:, 7]
    pcd = pc.detach()
    fx, fy = K[0, 0], K[1, 1]
    zeros = torch.zeros_like(pcd[:, 0])
    J = torch.stack([torch.stack([fx / pcd[:, 2], zeros, -fx * pcd[:, 0] / pcd[:, 2] ** 2], -1),
                     torch.stack([zeros, fy / pcd[:, 2], -fy * pcd[:, 1] / pcd[:, 2] ** 2], -1)], -2)
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
