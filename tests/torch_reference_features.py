"""The blend of per-Gaussian feature vectors by the dense float64 evaluator's weights (``torch_reference.dense_render``) --
what ``point_extra_features`` of the operator renders and differentiates (test helper).

Like ``torch_reference_depth``, this replays ``dense_render``'s compositing -- the same tile-membership mask, depth order,
1/255 cut, 0.99 straight-through clamp and 1e-4 early stop -- on the differentiable intermediates it returns, so that the
feature map shares one autograd graph with the image back to xyz and the 56 feature columns, and is differentiable in the
(N,C) features as well (rows gathered by ``aux["ids"]``)."""
import torch


def feature_map(aux, features, H, W, depth_scale=100.0):
    """F_p = sum_i w_i f_i per pixel (no normalisation), (H, W, C); ``aux`` from ``dense_render``, ``features`` (N, C)."""
    uv, z, opacity, radius = aux["uv"], aux["pc"][:, 2], aux["opacity"], aux["radius"]
    ca, cb, cc, rescale = aux["conic"].unbind(-1)
    dt = uv.dtype
    M = uv.shape[0]
    f = features[aux["ids"]].to(dt)
    C = f.shape[1]
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
    F = torch.zeros((H, W, C), dtype=dt)
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
        F = F + torch.where(blend[..., None], f[m][None, None, :] * w[..., None], torch.zeros_like(F))
        T = torch.where(blend, nT, T)
    return F
