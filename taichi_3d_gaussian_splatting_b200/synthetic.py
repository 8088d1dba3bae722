"""Synthetic scene generator ``S(N, seed)`` used by the parity tests and ``bench.py``.

The spec is SURVEY.md §8(d) / BASELINE.md §2: identity camera pose, fx = fy = 0.6·W, principal
point at the image centre; x~U(-4,4), y~U(-2.5,2.5), z~U(2,10); q~N(0,1)^4 normalised (xyzw);
log-scale ~ N(ln sigma_med, 0.5^2) per axis; opacity logit ~ U(-3,3); SH DC ~ N(0,1.5^2);
SH deg 3: the remaining 45 coefficients ~ N(0,0.2^2) (zeros for SH deg 0).
Feature row layout = the reference's 56-float row (GaussianPointCloudRasterisation.py:208-236).
"""
import math
from dataclasses import dataclass

import torch

from .Camera import CameraInfo


@dataclass
class SyntheticScene:
    point_cloud: torch.Tensor  # (N, 3) f32
    point_cloud_features: torch.Tensor  # (N, 56) f32
    point_invalid_mask: torch.Tensor  # (N,) i8
    point_object_id: torch.Tensor  # (N,) i32
    camera_info: CameraInfo
    q_pointcloud_camera: torch.Tensor  # (1, 4) xyzw
    t_pointcloud_camera: torch.Tensor  # (1, 3)

    def to(self, device) -> "SyntheticScene":
        ci = self.camera_info
        return SyntheticScene(
            self.point_cloud.to(device), self.point_cloud_features.to(device),
            self.point_invalid_mask.to(device), self.point_object_id.to(device),
            CameraInfo(ci.camera_intrinsics.to(device), ci.camera_height, ci.camera_width, ci.camera_id, ci.distortion,
                       ci.rolling_shutter, ci.motion_blur, ci.defocus),
            self.q_pointcloud_camera.to(device), self.t_pointcloud_camera.to(device))


def make_scene(num_points: int, height: int, width: int, sigma_med: float, seed: int,
               sh_degree: int = 3, yaw_degrees: float = 0.0) -> SyntheticScene:
    g = torch.Generator(device="cpu").manual_seed(seed)
    N = int(num_points)
    u = torch.rand((N, 3), generator=g, dtype=torch.float32)
    xyz = torch.stack([u[:, 0] * 8 - 4, u[:, 1] * 5 - 2.5, u[:, 2] * 8 + 2], dim=-1)
    q = torch.randn((N, 4), generator=g, dtype=torch.float32)
    q = q / q.norm(dim=-1, keepdim=True)
    s = torch.randn((N, 3), generator=g, dtype=torch.float32) * 0.5 + math.log(sigma_med)
    logit = torch.rand((N, 1), generator=g, dtype=torch.float32) * 6 - 3
    sh = torch.zeros((N, 3, 16), dtype=torch.float32)
    sh[:, :, 0] = torch.randn((N, 3), generator=g, dtype=torch.float32) * 1.5
    rest = torch.randn((N, 3, 15), generator=g, dtype=torch.float32) * 0.2
    if sh_degree > 0:
        n_rest = (sh_degree + 1) ** 2 - 1
        sh[:, :, 1:1 + n_rest] = rest[:, :, :n_rest]
    feats = torch.cat([q, s, logit, sh.reshape(N, 48)], dim=-1).contiguous()
    K = torch.tensor([[0.6 * width, 0.0, width / 2.0], [0.0, 0.6 * width, height / 2.0],
                      [0.0, 0.0, 1.0]], dtype=torch.float32)
    half = math.radians(yaw_degrees) / 2.0  # rotation about +y (down) of the camera in the scene
    q_pc = torch.tensor([[0.0, math.sin(half), 0.0, math.cos(half)]], dtype=torch.float32)
    t_pc = torch.zeros((1, 3), dtype=torch.float32)
    return SyntheticScene(
        point_cloud=xyz.contiguous(), point_cloud_features=feats,
        point_invalid_mask=torch.zeros((N,), dtype=torch.int8),
        point_object_id=torch.zeros((N,), dtype=torch.int32),
        camera_info=CameraInfo(camera_intrinsics=K, camera_height=height, camera_width=width, camera_id=0),
        q_pointcloud_camera=q_pc, t_pointcloud_camera=t_pc)


# BASELINE.md §2 configurations (reference multiple-of-16 rule applied to the image sizes)
CONFIGS = {
    "C1": dict(num_points=10_000, height=256, width=256, sigma_med=0.03, seed=0, sh_degree=0),
    "C2": dict(num_points=430_000, height=544, width=976, sigma_med=0.02, seed=1, sh_degree=3),
    "C3": dict(num_points=1_000_000, height=1072, width=1920, sigma_med=0.01, seed=2, sh_degree=3),
    "C3s": dict(num_points=1_000_000, height=1072, width=1920, sigma_med=0.02, seed=2, sh_degree=3),
    "C4": dict(num_points=2_100_000, height=1072, width=1920, sigma_med=0.01, seed=3, sh_degree=3),
}
C4_YAWS = (0.0, 5.0, -5.0, 10.0, -10.0, 15.0, -15.0, 20.0)


def make_panorama_scene(num_points: int, height: int, width: int, sigma_med: float, seed: int, sh_degree: int = 3,
                        radius: float = 4.0, yaw_degrees: float = 0.0, seam_fraction: float = 0.1,
                        pole_fraction: float = 0.05) -> SyntheticScene:
    """An equirectangular view (``LensDistortion("equirectangular", ())``, K of a full panorama) at the origin inside a
    shell of Gaussians: directions uniform on the sphere, distances radius * U(0.75, 1.25).  ``seam_fraction`` of the points
    lie within 10 degrees of longitude of the seam behind the camera (-z), ``pole_fraction`` within 10 degrees of a pole.
    Features as ``make_scene``."""
    from .Camera import LensDistortion
    g = torch.Generator(device="cpu").manual_seed(seed)
    N = int(num_points)
    d = torch.randn((N, 3), generator=g, dtype=torch.float64)
    d = d / d.norm(dim=-1, keepdim=True)
    n_seam, n_pole = int(N * seam_fraction), int(N * pole_fraction)
    if n_seam:  # longitude pi +- 10 degrees, latitude in +-60 degrees
        lon = math.pi + (torch.rand(n_seam, generator=g, dtype=torch.float64) * 2 - 1) * math.radians(10.0)
        lat = (torch.rand(n_seam, generator=g, dtype=torch.float64) * 2 - 1) * math.radians(60.0)
        d[:n_seam] = torch.stack([torch.cos(lat) * torch.sin(lon), torch.sin(lat), torch.cos(lat) * torch.cos(lon)], -1)
    if n_pole:  # within 10 degrees of +y or -y
        lon = torch.rand(n_pole, generator=g, dtype=torch.float64) * 2 * math.pi
        colat = torch.rand(n_pole, generator=g, dtype=torch.float64) * math.radians(10.0)
        sign = torch.where(torch.rand(n_pole, generator=g) < 0.5, -1.0, 1.0).to(torch.float64)
        d[n_seam:n_seam + n_pole] = torch.stack([torch.sin(colat) * torch.sin(lon), sign * torch.cos(colat),
                                                 torch.sin(colat) * torch.cos(lon)], -1)
    dist = radius * (0.75 + 0.5 * torch.rand((N, 1), generator=g, dtype=torch.float64))
    xyz = (d * dist).to(torch.float32)
    q = torch.randn((N, 4), generator=g, dtype=torch.float32)
    q = q / q.norm(dim=-1, keepdim=True)
    s = torch.randn((N, 3), generator=g, dtype=torch.float32) * 0.5 + math.log(sigma_med)
    logit = torch.rand((N, 1), generator=g, dtype=torch.float32) * 6 - 3
    sh = torch.zeros((N, 3, 16), dtype=torch.float32)
    sh[:, :, 0] = torch.randn((N, 3), generator=g, dtype=torch.float32) * 1.5
    rest = torch.randn((N, 3, 15), generator=g, dtype=torch.float32) * 0.2
    if sh_degree > 0:
        n_rest = (sh_degree + 1) ** 2 - 1
        sh[:, :, 1:1 + n_rest] = rest[:, :, :n_rest]
    feats = torch.cat([q, s, logit, sh.reshape(N, 48)], dim=-1).contiguous()
    half = math.radians(yaw_degrees) / 2.0
    return SyntheticScene(
        point_cloud=xyz.contiguous(), point_cloud_features=feats,
        point_invalid_mask=torch.zeros((N,), dtype=torch.int8), point_object_id=torch.zeros((N,), dtype=torch.int32),
        camera_info=CameraInfo(camera_intrinsics=LensDistortion.equirectangular_intrinsics(width, height),
                               camera_height=height, camera_width=width, camera_id=0,
                               distortion=LensDistortion("equirectangular", ())),
        q_pointcloud_camera=torch.tensor([[0.0, math.sin(half), 0.0, math.cos(half)]], dtype=torch.float32),
        t_pointcloud_camera=torch.zeros((1, 3), dtype=torch.float32))
