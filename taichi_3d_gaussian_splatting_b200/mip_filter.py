"""3D smoothing filter (Mip-Splatting, Yu et al., CVPR 2024): every Gaussian is convolved in world space with an isotropic
Gaussian of std sigma_i, the finest sampling interval of the training views that see it, so that a trained scene holds no
frequency those views did not constrain.  Definition in ``include/gsb200.h``.

``compute_filter_3d`` computes sigma from the training views (``gsb200_filter3d_from_views`` on CUDA tensors, the same rule on
the host for CPU tensors).  The rasteriser takes it as ``point_filter_3d`` and renders the filtered Gaussians without changing
the stored rows; ``bake_filter_3d`` writes the filtered scales and opacities into a copy of the rows, for export and tests.
"""
import ctypes
import math
from typing import Sequence, Tuple

import numpy as np
import torch

from . import _lib

DEFAULT_VARIANCE = 0.2  # the paper's value, in pixels^2 at the finest view
VIEW_MARGIN = 0.15      # a view sees a point projected up to 15 % of the image size outside it


def _pose_matrices(q: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
    """(n, 3, 4) float32 [R | t'] of the camera-from-scene maps, bit for bit as the rasteriser's pose kernel forms them (q
    conjugated, normalised for the translation only): numpy float32 ufuncs, one rounding per operation in the kernel's order
    (torch's CPU kernels may contract a multiply and an add into one fused operation)."""
    f32 = np.float32
    q = q.detach().cpu().numpy().astype(f32)
    t = t.detach().cpu().numpy().astype(f32)
    qi = [-q[:, 0], -q[:, 1], -q[:, 2], q[:, 3]]
    n = np.sqrt(((qi[0] * qi[0] + qi[1] * qi[1]) + qi[2] * qi[2]) + qi[3] * qi[3])
    qn = [c / n for c in qi]

    def mul(a, b):
        x0, y0, z0, w0 = a
        x1, y1, z1, w1 = b
        return [w0 * x1 + x0 * w1 + y0 * z1 - z0 * y1, w0 * y1 - x0 * z1 + y0 * w1 + z0 * x1,
                w0 * z1 + x0 * y1 - y0 * x1 + z0 * w1, w0 * w1 - x0 * x1 - y0 * y1 - z0 * z1]

    v = [t[:, 0], t[:, 1], t[:, 2], np.zeros_like(t[:, 0])]
    rot = mul(mul(qn, v), [-qn[0], -qn[1], -qn[2], qn[3]])
    x, y, z, w = qi
    xx, yy, zz, xy, xz, yz, wx, wy, wz = x * x, y * y, z * z, x * y, x * z, y * z, w * x, w * y, w * z
    one, two = f32(1), f32(2)
    rows = [[one - two * (yy + zz), two * (xy - wz), two * (xz + wy), -rot[0]],
            [two * (xy + wz), one - two * (xx + zz), two * (yz - wx), -rot[1]],
            [two * (xz - wy), two * (yz + wx), one - two * (xx + yy), -rot[2]]]
    return torch.from_numpy(np.stack([np.stack(r, axis=1) for r in rows], axis=1).astype(f32))


def _filter_rule(xyz, invalid, obj, poses, K, sizes, near_plane, variance):
    """The rule of ``gsb200_filter3d_from_views`` on the host (the reference form of the kernel, CPU tensors): numpy float32
    ufuncs with the kernel's operation order, so the result is the kernel's bit for bit.  A row whose object id is outside
    [0, objects) matches no view, as in the kernel."""
    f32 = np.float32
    xyz = xyz.detach().cpu().numpy().astype(f32)
    valid = invalid.detach().cpu().numpy() == 0
    obj = obj.detach().cpu().numpy().astype(np.int64)
    poses, K = poses.numpy().astype(f32), K.detach().cpu().numpy().astype(f32)
    N, V = xyz.shape[0], K.shape[0]
    n_obj = poses.shape[0] // V
    has_obj = (obj >= 0) & (obj < n_obj)
    ob = np.where(has_obj, obj, 0)
    d_min = np.full(N, np.inf, f32)
    seen = np.zeros(N, bool)
    x, y, z = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    for v in range(V):
        T = poses.reshape(V, n_obj, 3, 4)[v][ob]  # (N, 3, 4)
        pc = [((T[:, r, 0] * x + T[:, r, 1] * y) + T[:, r, 2] * z) + T[:, r, 3] * f32(1) for r in range(3)]
        k = K[v].reshape(-1)
        f = np.fmax(k[0], k[4])  # as fmaxf: a NaN entry is ignored
        with np.errstate(divide="ignore", invalid="ignore"):
            u = ((k[0] * pc[0] + k[1] * pc[1]) + k[2] * pc[2]) / pc[2]
            vv = ((k[3] * pc[0] + k[4] * pc[1]) + k[5] * pc[2]) / pc[2]
            d = pc[2] / f
        Wf, Hf = f32(sizes[v][0]), f32(sizes[v][1])
        sees = valid & has_obj & (pc[2] > f32(near_plane)) & (f > 0) & (u >= f32(-0.15) * Wf) & (u <= f32(1.15) * Wf) & \
            (vv >= f32(-0.15) * Hf) & (vv <= f32(1.15) * Hf)
        d_min = np.where(sees, np.fmin(d_min, d), d_min)
        seen |= sees
    sqrt_var = np.sqrt(f32(variance))
    d_max = d_min[seen].max() if seen.any() else f32(0)
    out = np.where(valid, sqrt_var * np.where(seen, d_min, d_max), f32(0)).astype(f32)
    return torch.from_numpy(out)


def compute_filter_3d(point_cloud: torch.Tensor, point_invalid_mask: torch.Tensor, point_object_id: torch.Tensor,
                      views: Sequence[Tuple[torch.Tensor, torch.Tensor, object]], near_plane: float,
                      variance: float = DEFAULT_VARIANCE) -> torch.Tensor:
    """The (N,) float32 3D filter std of every row, on the scene's device.  ``views``: (q_pointcloud_camera (K, 4),
    t_pointcloud_camera (K, 3), camera_info) of every training view at FULL resolution (``camera_info`` gives
    ``camera_intrinsics``, ``camera_width`` and ``camera_height``; a lens or rolling shutter is ignored: the pinhole test at
    the mid-readout pose is an approximation for those views).  ``near_plane``: the rasteriser's.  ``variance``: in pixels^2
    at the finest view.  CUDA tensors run ``gsb200_filter3d_from_views``; CPU tensors the same rule on the host, bit for bit.
    ``ValueError`` unless the point cloud is float32 (N, 3), the mask int8 (N,) and the object ids int32 (N,), all on one
    device."""
    if len(views) < 1:
        raise ValueError("compute_filter_3d needs at least one view")
    if any(getattr(getattr(ci, "distortion", None), "model", None) == "orthographic" for _, _, ci in views):
        # the rule's frustum and sampling rate (f / z) are the pinhole's
        raise ValueError("compute_filter_3d does not take orthographic views")
    if not (math.isfinite(near_plane) and near_plane >= 0 and math.isfinite(variance) and variance >= 0):
        raise ValueError(f"near_plane and variance must be finite and >= 0, got {near_plane}, {variance}")
    device = point_cloud.device
    n_obj = views[0][0].shape[0]
    if any(q.shape[0] != n_obj or t.shape[0] != n_obj for q, t, _ in views):
        raise ValueError("every view must give the pose of every object")
    q = torch.cat([q.detach().reshape(-1, 4) for q, _, _ in views]).to(device=device, dtype=torch.float32).contiguous()
    t = torch.cat([t.detach().reshape(-1, 3) for _, t, _ in views]).to(device=device, dtype=torch.float32).contiguous()
    K = torch.stack([ci.camera_intrinsics.detach().to(device=device, dtype=torch.float32).reshape(3, 3)
                     for _, _, ci in views]).contiguous()
    sizes = torch.tensor([[int(ci.camera_width), int(ci.camera_height)] for _, _, ci in views], dtype=torch.int32)
    xyz = point_cloud.detach().contiguous()
    N = xyz.shape[0]
    for name, x, dtype, shape in (("point_cloud", xyz, torch.float32, (N, 3)),
                                  ("point_invalid_mask", point_invalid_mask, torch.int8, (N,)),
                                  ("point_object_id", point_object_id, torch.int32, (N,))):
        if x.dtype != dtype or x.device != device or tuple(x.shape) != shape:
            raise ValueError(f"{name} must be a {dtype} {shape} tensor on {device}, got {x.dtype} {tuple(x.shape)} "
                             f"on {x.device}")
    if not xyz.is_cuda:
        return _filter_rule(xyz, point_invalid_mask, point_object_id, _pose_matrices(q, t), K, sizes, float(near_plane),
                            float(variance))
    lib = _lib.load()
    V = len(views)
    sizes = sizes.to(device)
    out = torch.empty((N,), dtype=torch.float32, device=device)
    temp_bytes = int(lib.gsb200_filter3d_temp_bytes(V, n_obj))
    temp = torch.empty((temp_bytes,), dtype=torch.uint8, device=device)
    mask = point_invalid_mask.contiguous()
    obj = point_object_id.contiguous()
    with torch.cuda.device(device):
        args = _lib.GsbFilter3dViewsArgs(
            num_points=N, pointcloud=xyz.data_ptr(), point_invalid_mask=mask.data_ptr(), point_object_id=obj.data_ptr(),
            num_objects=n_obj, num_views=V, q_pointcloud_camera=q.data_ptr(), t_pointcloud_camera=t.data_ptr(),
            camera_intrinsics=K.data_ptr(), camera_size=sizes.data_ptr(), near_plane=float(near_plane),
            variance=float(variance), filter3d=out.data_ptr(), temp=temp.data_ptr(), temp_bytes=temp_bytes,
            stream=torch.cuda.current_stream(device).cuda_stream)
        _lib.check(lib.gsb200_filter3d_from_views(ctypes.byref(args)), "gsb200_filter3d_from_views")
    return out


def bake_filter_3d(features: torch.Tensor, filter_3d: torch.Tensor) -> torch.Tensor:
    """A copy of the (N, 56) rows with the filtered log-scales log(s^) and the filtered opacity logit logit(o c) written in
    (computed in float64, returned in the rows' dtype): the unfiltered rasteriser renders these rows as the filtered one
    renders the originals.  Rows with sigma = 0 (or NaN / negative sigma, read as 0) are returned unchanged."""
    out = features.detach().clone()
    f = features.detach().to(torch.float64)
    sigma = torch.nan_to_num(filter_3d.detach().to(torch.float64), nan=0.0).clamp_min(0.0)
    s2 = (sigma * sigma)[:, None]
    e = torch.exp(f[:, 4:7]) ** 2
    eh = e + s2
    c = torch.sqrt(torch.prod(e / eh, dim=1))
    o = torch.sigmoid(f[:, 7]) * c
    on = (sigma > 0) & (s2[:, 0] > 0)
    out[on, 4:7] = (0.5 * torch.log(eh[on])).to(out.dtype)
    out[on, 7] = torch.log(o[on] / (1 - o[on])).to(out.dtype)
    return out
