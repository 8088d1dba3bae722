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


# The raised blocks of make_aerial_scene: (x0, x1, y0, y1, height) as fractions of the ground's width (x0..y1) and of the
# camera's height above the ground (height).  They do not overlap.
AERIAL_BLOCKS = ((-0.30, -0.10, -0.25, 0.05, 0.20), (0.10, 0.35, 0.10, 0.30, 0.35), (0.05, 0.25, -0.40, -0.20, 0.12))


def aerial_height(x: torch.Tensor, y: torch.Tensor, ground_width: float, altitude: float) -> torch.Tensor:
    """The surface height of make_aerial_scene at scene (x, y): a block's height on its top, 0 elsewhere."""
    h = torch.zeros_like(x)
    for x0, x1, y0, y1, hb in AERIAL_BLOCKS:
        inside = (x >= x0 * ground_width) & (x < x1 * ground_width) & (y >= y0 * ground_width) & (y < y1 * ground_width)
        h = torch.where(inside, torch.full_like(x, hb * altitude), h)
    return h


def aerial_texture(x: torch.Tensor, y: torch.Tensor, ground_width: float) -> torch.Tensor:
    """(..., 3) colours in [0.15, 0.85] of make_aerial_scene's ground at scene (x, y): smooth stripes of 1/8 and 1/6 of the
    ground's width, so that a render at a few pixels per stripe period resolves them."""
    a = 2.0 * math.pi * x / (ground_width / 8.0)
    b = 2.0 * math.pi * y / (ground_width / 6.0)
    return torch.stack([0.5 + 0.35 * torch.sin(a), 0.5 + 0.35 * torch.cos(b), 0.5 + 0.35 * torch.sin(a) * torch.cos(b)], -1)


def make_aerial_scene(num_points: int, height: int, width: int, seed: int, pixel_size: float = 0.01,
                      altitude: float = 5.0) -> SyntheticScene:
    """A drone-survey-like scene for orthographic views: a textured ground plane z = 0 (scene up = +z) with the raised
    blocks of ``AERIAL_BLOCKS``, made of flat, nearly opaque Gaussians at random positions on the visible surface (the blocks'
    tops; their sides are not drawn), coloured by ``aerial_texture`` through the SH DC term alone.  The ground is 10 % wider
    than the image's footprint at ``pixel_size`` scene units per pixel.  The camera is the nadir orthographic view of
    ``Camera.orthographic_view`` at (0, 0, ``altitude``) with +y toward the top of the image, so pixel (u, v) sees scene
    x = (u - W/2) pixel_size, y = (H/2 - v) pixel_size, and the height under it is ``altitude`` - depth."""
    from .Camera import orthographic_view
    g = torch.Generator(device="cpu").manual_seed(seed)
    N = int(num_points)
    gw, gh = 1.1 * width * pixel_size, 1.1 * height * pixel_size
    u = torch.rand((N, 2), generator=g, dtype=torch.float32)
    x, y = (u[:, 0] - 0.5) * gw, (u[:, 1] - 0.5) * gh
    z = aerial_height(x, y, gw, altitude)
    xyz = torch.stack([x, y, z], -1)
    spacing = math.sqrt(gw * gh / max(N, 1))
    q = torch.zeros((N, 4), dtype=torch.float32)
    q[:, 3] = 1.0
    s = torch.empty((N, 3), dtype=torch.float32)
    s[:, 0:2] = math.log(0.7 * spacing)
    s[:, 2] = math.log(0.1 * spacing)
    logit = torch.full((N, 1), 4.0)
    rgb = aerial_texture(x, y, gw)
    sh = torch.zeros((N, 3, 16), dtype=torch.float32)
    sh[:, :, 0] = torch.logit(rgb) / 0.28209479177387814
    feats = torch.cat([q, s, logit, sh.reshape(N, 48)], dim=-1).contiguous()
    q_pc, t_pc, ci = orthographic_view((0.0, 0.0, altitude), (0.0, 0.0, -1.0), (0.0, 1.0, 0.0), width, height, pixel_size)
    return SyntheticScene(
        point_cloud=xyz.contiguous(), point_cloud_features=feats,
        point_invalid_mask=torch.zeros((N,), dtype=torch.int8), point_object_id=torch.zeros((N,), dtype=torch.int32),
        camera_info=ci, q_pointcloud_camera=q_pc, t_pointcloud_camera=t_pc)
