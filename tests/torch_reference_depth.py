"""The depth map of the dense float64 evaluator (``torch_reference.dense_render``) made differentiable in each splat's
camera-space depth z as well -- what ``differentiable_depth=True`` of the operator differentiates (test helper).

``dense_render`` composites the depth with z detached (nothing differentiates the reference's depth).  This module replays
the same compositing -- the same tile-membership mask, depth order, 1/255 cut, 0.99 straight-through clamp and 1e-4
early stop -- on the differentiable intermediates ``dense_render`` returns (uv, conic, opacity, camera-space position),
so the image and this depth map share one autograd graph back to xyz and the features."""
import torch


def differentiable_depth(aux, H, W, depth_scale=100.0):
    """D = sum w z / max(sum w, 1e-6) per pixel, differentiable through w (uv, conic, opacity) and z; ``aux`` from
    ``dense_render``.  Also returns the blended-pair count, which must equal ``aux["count"]``."""
    uv, z, opacity, radius = aux["uv"], aux["pc"][:, 2], aux["opacity"], aux["radius"]
    ca, cb, cc, rescale = aux["conic"].unbind(-1)
    dt = uv.dtype
    M = uv.shape[0]
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
    D = torch.zeros((H, W), dtype=dt)
    Wt = torch.zeros((H, W), dtype=dt)
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
        D = D + torch.where(blend, z[m] * w, torch.zeros_like(D))
        Wt = Wt + torch.where(blend, w, torch.zeros_like(Wt))
        cnt = cnt + blend.to(torch.int32)
        T = torch.where(blend, nT, T)
    return D / torch.clamp(Wt, min=1e-6), cnt
