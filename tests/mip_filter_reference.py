"""TEST HELPER: the 3D smoothing filter (include/gsb200.h) restated with explicit loops -- the application in float64 and the
views rule in float32 with the kernel's operation order -- plus a differentiable torch bake and an oracle-backed module
that renders through it, so that the trainer harness can run with the filter on the CPU."""
import math

import numpy as np
import torch

from taichi_3d_gaussian_splatting_b200.Camera import CameraInfo

from oracle_module import OracleRasterisationModule


def bake_reference(features, sigma):
    """(N, 56) float64: per row, log s^_j = 0.5 log(exp(s_j)^2 + sigma^2) and logit(o c); sigma NaN / <= 0: unchanged."""
    f = np.array(features, np.float64)
    out = f.copy()
    for i in range(f.shape[0]):
        sg = float(sigma[i])
        if not (sg > 0.0):
            continue
        c2 = 1.0
        for j in range(3):
            e = math.exp(f[i, 4 + j]) ** 2
            eh = e + sg * sg
            c2 *= e / eh
            out[i, 4 + j] = 0.5 * math.log(eh)
        o = 1.0 / (1.0 + math.exp(-f[i, 7])) * math.sqrt(c2)
        out[i, 7] = math.log(o / (1.0 - o))
    return out


def bake_torch(features, sigma):
    """The bake as differentiable torch ops in the rows' dtype (sigma is a constant): the unfiltered operator on these rows
    renders what the filtered operator renders on the originals."""
    sg = torch.nan_to_num(sigma.detach(), nan=0.0).clamp_min(0.0).to(features.dtype)
    s2 = (sg * sg)[:, None]
    on = (s2[:, 0] > 0)[:, None]
    e = torch.exp(features[:, 4:7]) ** 2
    eh = e + s2
    s_hat = torch.where(on, 0.5 * torch.log(torch.where(on, eh, torch.ones_like(eh))), features[:, 4:7])
    c = torch.sqrt(torch.prod(torch.where(on, e / eh, torch.ones_like(e)), dim=1))
    o = torch.sigmoid(features[:, 7]) * c
    logit = torch.where(on[:, 0], torch.log(o) - torch.log1p(-o), features[:, 7])
    return torch.cat([features[:, 0:4], s_hat, logit[:, None], features[:, 8:]], dim=1)


def filter_reference(xyz, invalid, obj, poses, K, sizes, near_plane, variance):
    """The views rule with explicit loops.  poses: (V, n_obj, 3, 4) float32 camera-from-scene maps (as the pose kernel
    forms them); K (V, 3, 3); sizes (V, 2) {W, H}.  float32 arithmetic in the kernel's order for every decision."""
    f32 = np.float32
    xyz, poses, K = np.asarray(xyz, f32), np.asarray(poses, f32), np.asarray(K, f32)
    N, V = xyz.shape[0], K.shape[0]
    d = np.full(N, np.inf, f32)
    seen = np.zeros(N, bool)
    for i in range(N):
        if invalid[i] != 0:
            continue
        x, y, z = xyz[i]
        if not 0 <= obj[i] < poses.shape[1]:  # an object id outside the scene's objects matches no view
            continue
        for v in range(V):
            T = poses[v, obj[i]]
            pc = [((T[r, 0] * x + T[r, 1] * y) + T[r, 2] * z) + T[r, 3] * f32(1.0) for r in range(3)]
            k = K[v].reshape(-1)
            f = np.fmax(k[0], k[4])  # fmaxf: a NaN entry is ignored
            if not (pc[2] > f32(near_plane) and f > 0):
                continue
            u = ((k[0] * pc[0] + k[1] * pc[1]) + k[2] * pc[2]) / pc[2]
            vv = ((k[3] * pc[0] + k[4] * pc[1]) + k[5] * pc[2]) / pc[2]
            Wf, Hf = f32(sizes[v][0]), f32(sizes[v][1])
            if f32(-0.15) * Wf <= u <= f32(1.15) * Wf and f32(-0.15) * Hf <= vv <= f32(1.15) * Hf:
                d[i] = min(d[i], pc[2] / f)
                seen[i] = True
    d_max = d[seen].max() if seen.any() else f32(0.0)
    out = np.zeros(N, f32)
    sv = np.sqrt(f32(variance))
    for i in range(N):
        if invalid[i] == 0:
            out[i] = sv * (d[i] if seen[i] else d_max)
    return out


def random_views(V, n_obj, g, W=320, H=240):
    """V views of n_obj objects: random yaw / pitch and translation, focal lengths between 0.4 W and 1.2 W."""
    views = []
    for _ in range(V):
        a = (torch.rand(3, generator=g) - 0.5) * 0.6
        q = torch.stack([torch.cat([a[:2] * torch.rand(1, generator=g), a[2:] * 0.2,
                                    torch.ones(1)]) for _ in range(n_obj)])
        q = q / q.norm(dim=1, keepdim=True) * (1.0 + 0.05 * torch.rand((n_obj, 1), generator=g))
        t = (torch.rand((n_obj, 3), generator=g) - 0.5) * 2.0
        f = float(W) * (0.4 + 0.8 * float(torch.rand(1, generator=g)))
        K = torch.tensor([[f, 0.0, W / 2.0], [0.0, f * 0.97, H / 2.0], [0.0, 0.0, 1.0]])
        views.append((q.float().contiguous(), t.float().contiguous(), CameraInfo(K, H, W, 0)))
    return views


class FilteredOracleModule(OracleRasterisationModule):
    """The oracle module that takes ``point_filter_3d`` and renders the baked rows (autograd through the bake)."""
    calls = []  # (filter or None) of every forward, for the tests

    def forward(self, inp, point_filter_3d=None):
        FilteredOracleModule.calls.append(None if point_filter_3d is None else point_filter_3d.clone())
        if point_filter_3d is None:
            return super().forward(inp)
        baked = bake_torch(inp.point_cloud_features, point_filter_3d).contiguous()
        return super().forward(type(inp)(point_cloud=inp.point_cloud, point_cloud_features=baked,
                                         point_object_id=inp.point_object_id, point_invalid_mask=inp.point_invalid_mask,
                                         camera_info=inp.camera_info, q_pointcloud_camera=inp.q_pointcloud_camera,
                                         t_pointcloud_camera=inp.t_pointcloud_camera, color_max_sh_band=inp.color_max_sh_band))
