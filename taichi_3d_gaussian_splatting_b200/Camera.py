"""Camera dataclasses -- the argument types of the rasteriser operator.

Mirrors the reference's ``taichi_3d_gaussian_splatting/Camera.py:7-21`` (``CameraInfo`` is an
argument of ``GaussianPointCloudRasterisationInput``; ``CameraView`` is imported beside it at
GaussianPointCloudRasterisation.py:4).  ``LensDistortion`` and ``CameraInfo.distortion`` are an extension: the reference
projects through a pinhole only.  ``RollingShutter`` and ``CameraInfo.rolling_shutter`` are an extension as well: the reference
projects every row with one global-shutter pose.  So are ``MotionBlur`` and ``CameraInfo.motion_blur``: the reference renders every
view as if the shutter were instantaneous; and ``Defocus`` and ``CameraInfo.defocus``: the reference renders through an ideal
pinhole, sharp at every depth.  ``LensDistortion("orthographic", ())`` and ``orthographic_view`` are an extension too: the
reference has no parallel projection.
"""
import math
from dataclasses import dataclass
from typing import Optional, Sequence, Tuple

import torch

_LENS_COEFFICIENTS = {"opencv": 5, "fisheye": 4, "equirectangular": 0, "orthographic": 0}


@dataclass(frozen=True)
class LensDistortion:
    """A lens between the camera-frame point and K (definition in ``include/gsb200.h``), as host floats so that rendering a
    view reads nothing back from the device.

    ``model``: ``"opencv"`` -- coefficients ``(k1, k2, p1, p2, k3)`` in OpenCV's ``distCoeffs`` order (COLMAP
    ``SIMPLE_RADIAL``, ``RADIAL``, ``OPENCV``) -- or ``"fisheye"`` -- ``(k1, k2, k3, k4)`` of the equidistant model (COLMAP
    ``OPENCV_FISHEYE``, ``cv2.fisheye``).  The coefficients act on the normalised image plane (x/z, y/z), so resizing or
    cropping an image changes K but not them.

    ``"equirectangular"`` (no coefficients) is the 360-degree panorama of Insta360, Ricoh Theta, GoPro Max and drone panorama
    modes: u = fx atan2(x, z) + cx (wrapped into [0, W)), v = fy atan2(y, sqrt(x^2 + z^2)) + cy, with 2 pi fx = W (definition in
    ``include/gsb200.h``; K from ``equirectangular_intrinsics``).  It renders and trains the point gradients only: no pose,
    intrinsics or lens gradient, rolling shutter, motion blur, defocus, 3D filter or view-parallel exchange.

    ``"orthographic"`` (no coefficients) is the parallel projection of orthophotos, orthorectified aerial tiles, satellite
    crops and CAD renders: u = K00 x + K01 y + K02, v = K10 x + K11 y + K12 of the camera-frame point, no divide, so fx and fy
    are pixels per scene unit (definition in ``include/gsb200.h``; K from ``orthographic_intrinsics``).  Depth is z, and the SH
    colour is seen along the camera's forward axis.  It renders and trains the point, pose and intrinsics gradients, with
    depth, alpha, features and the 3D filter (the filter without camera gradients); no lens gradient, rolling shutter, motion
    blur, defocus or view-parallel exchange."""
    model: str
    coefficients: Tuple[float, ...]

    def __post_init__(self):
        if self.model not in _LENS_COEFFICIENTS:
            raise ValueError(f"lens model must be one of {tuple(_LENS_COEFFICIENTS)}, got {self.model!r}")
        co = tuple(float(v) for v in self.coefficients)
        if len(co) != _LENS_COEFFICIENTS[self.model]:
            raise ValueError(f"the {self.model} lens takes {_LENS_COEFFICIENTS[self.model]} coefficients, got {len(co)}")
        if not all(math.isfinite(v) for v in co):
            raise ValueError(f"lens coefficients must be finite, got {co}")
        object.__setattr__(self, "coefficients", co)

    @staticmethod
    def equirectangular_intrinsics(width: int, height: int) -> torch.Tensor:
        """K (3,3) float32 of a full equirectangular panorama: fx = W / 2pi, fy = H / pi, (cx, cy) = (W / 2, H / 2), so the image
        spans 360 x 180 degrees and its centre looks along +z."""
        w, h = int(width), int(height)
        if w <= 0 or h <= 0:
            raise ValueError(f"width and height must be positive, got {width} x {height}")
        return torch.tensor([[w / (2.0 * math.pi), 0.0, w / 2.0], [0.0, h / math.pi, h / 2.0], [0.0, 0.0, 1.0]],
                            dtype=torch.float32)

    @staticmethod
    def orthographic_intrinsics(width: int, height: int, pixel_size: float) -> torch.Tensor:
        """K (3,3) float32 of an orthographic view: fx = fy = 1 / pixel_size (pixels per scene unit; ``pixel_size`` is the
        ground sampling distance of an orthophoto) and the principal point at the image centre."""
        w, h, d = int(width), int(height), float(pixel_size)
        if w <= 0 or h <= 0:
            raise ValueError(f"width and height must be positive, got {width} x {height}")
        if not (math.isfinite(d) and d > 0.0):
            raise ValueError(f"pixel_size must be finite and > 0, got {pixel_size}")
        return torch.tensor([[1.0 / d, 0.0, w / 2.0], [0.0, 1.0 / d, h / 2.0], [0.0, 0.0, 1.0]], dtype=torch.float32)

    @staticmethod
    def from_colmap(model_name: str, params: Sequence[float]) -> Tuple[torch.Tensor, Optional["LensDistortion"]]:
        """(K (3,3) float32, lens or None) of a COLMAP camera: ``SIMPLE_PINHOLE`` (f cx cy), ``PINHOLE`` (fx fy cx cy),
        ``SIMPLE_RADIAL`` (f cx cy k), ``RADIAL`` (f cx cy k1 k2), ``OPENCV`` (fx fy cx cy k1 k2 p1 p2) and
        ``OPENCV_FISHEYE`` (fx fy cx cy k1 k2 k3 k4).  ``ValueError`` for any other model or a wrong parameter count."""
        counts = {"SIMPLE_PINHOLE": 3, "PINHOLE": 4, "SIMPLE_RADIAL": 4, "RADIAL": 5, "OPENCV": 8, "OPENCV_FISHEYE": 8}
        if model_name not in counts:
            raise ValueError(f"unsupported COLMAP camera model {model_name!r}: expected one of {tuple(counts)}")
        p = [float(v) for v in params]
        if len(p) != counts[model_name]:
            raise ValueError(f"COLMAP {model_name} has {counts[model_name]} parameters, got {len(p)}")
        if model_name in ("SIMPLE_PINHOLE", "SIMPLE_RADIAL", "RADIAL"):
            fx = fy = p[0]
            cx, cy, rest = p[1], p[2], p[3:]
        else:
            fx, fy, cx, cy, rest = p[0], p[1], p[2], p[3], p[4:]
        K = torch.tensor([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]], dtype=torch.float32)
        if model_name == "SIMPLE_RADIAL":
            return K, LensDistortion("opencv", (rest[0], 0.0, 0.0, 0.0, 0.0))
        if model_name == "RADIAL":
            return K, LensDistortion("opencv", (rest[0], rest[1], 0.0, 0.0, 0.0))
        if model_name == "OPENCV":
            return K, LensDistortion("opencv", tuple(rest) + (0.0,))
        if model_name == "OPENCV_FISHEYE":
            return K, LensDistortion("fisheye", tuple(rest))
        return K, None


@dataclass(frozen=True)
class RollingShutter:
    """The motion of a rolling-shutter view (definition in ``include/gsb200.h``), as host floats: ``linear`` = v (scene
    units) and ``angular`` = w (radians), the apparent motion of the scene in the camera frame over one full readout, top row
    to bottom row.  The view's pose is the pose at mid-readout.  Row time is normalised by the image height, so resizing or
    cropping an image keeps the motion."""
    linear: Tuple[float, float, float]
    angular: Tuple[float, float, float]

    def __post_init__(self):
        for name in ("linear", "angular"):
            v = tuple(float(x) for x in getattr(self, name))
            if len(v) != 3:
                raise ValueError(f"rolling-shutter {name} motion takes 3 values, got {len(v)}")
            if not all(math.isfinite(x) for x in v):
                raise ValueError(f"rolling-shutter {name} motion must be finite, got {v}")
            object.__setattr__(self, name, v)

    @staticmethod
    def from_camera_velocity(linear_velocity: Sequence[float], angular_velocity: Sequence[float],
                             readout_time: float) -> "RollingShutter":
        """The motion of a camera moving at ``linear_velocity`` (scene units/s) and ``angular_velocity`` (rad/s), both in
        the camera's own frame (what visual-inertial odometry and ARKit report), read out top to bottom in ``readout_time``
        seconds: a static scene moves the other way in the camera frame, v = -T u and w = -T w_c."""
        T = float(readout_time)
        if not (math.isfinite(T) and T >= 0.0):
            raise ValueError(f"readout_time must be finite and >= 0, got {readout_time}")
        return RollingShutter(tuple(-T * float(x) for x in linear_velocity), tuple(-T * float(x) for x in angular_velocity))

    @property
    def motion(self) -> Tuple[float, ...]:
        """(v, w) as six floats, the order of ``GsbRollingShutterArgs::motion``."""
        return self.linear + self.angular


@dataclass(frozen=True)
class MotionBlur:
    """The exposure motion of a blurred view (definition in ``include/gsb200.h``), as host floats: ``linear`` = v (scene
    units) and ``angular`` = w (radians), the apparent motion of the scene in the camera frame over the whole exposure, in the
    convention of ``RollingShutter``.  The view's pose is the pose at mid-exposure.

    Two properties of the model: only +-m is observable (the blur depends on d d^T, so m and -m render the same), and the
    blur's gradient with respect to m vanishes at m = 0, so refining it needs a non-zero start (from visual-inertial
    odometry through ``from_camera_velocity``, or from neighbouring frames through ``between_poses``)."""
    linear: Tuple[float, float, float]
    angular: Tuple[float, float, float]

    def __post_init__(self):
        for name in ("linear", "angular"):
            v = tuple(float(x) for x in getattr(self, name))
            if len(v) != 3:
                raise ValueError(f"motion-blur {name} motion takes 3 values, got {len(v)}")
            if not all(math.isfinite(x) for x in v):
                raise ValueError(f"motion-blur {name} motion must be finite, got {v}")
            object.__setattr__(self, name, v)

    @staticmethod
    def from_camera_velocity(linear_velocity: Sequence[float], angular_velocity: Sequence[float],
                             exposure_time: float) -> "MotionBlur":
        """The exposure motion of a camera moving at ``linear_velocity`` (scene units/s) and ``angular_velocity`` (rad/s),
        both in the camera's own frame (what visual-inertial odometry and ARKit report), with the shutter open for
        ``exposure_time`` seconds: a static scene moves the other way in the camera frame, v = -T u and w = -T w_c."""
        T = float(exposure_time)
        if not (math.isfinite(T) and T >= 0.0):
            raise ValueError(f"exposure_time must be finite and >= 0, got {exposure_time}")
        return MotionBlur(tuple(-T * float(x) for x in linear_velocity), tuple(-T * float(x) for x in angular_velocity))

    @staticmethod
    def between_poses(T_before: torch.Tensor, T_after: torch.Tensor, fraction: float) -> "MotionBlur":
        """The exposure motion of a view between two frames of a video at constant velocity, ``fraction`` = exposure time
        / frame interval.  ``T_before`` and ``T_after`` are the 4x4 camera -> scene transforms (``CameraView.
        T_pointcloud_camera``) of the earlier and the later frame.  A = T_after^-1 T_before = [R_A | t_A] maps camera-frame
        points of the earlier frame to the later one, and the motion is (fraction t_A, fraction log R_A): exact for this
        model's motion pc(t) = exp(t [w]x) pc + t v at constant velocity."""
        f = float(fraction)
        if not (math.isfinite(f) and f >= 0.0):
            raise ValueError(f"fraction must be finite and >= 0, got {fraction}")
        Tb = torch.as_tensor(T_before, dtype=torch.float64).cpu()
        Ta = torch.as_tensor(T_after, dtype=torch.float64).cpu()
        if Tb.shape != (4, 4) or Ta.shape != (4, 4):
            raise ValueError(f"T_before and T_after must be 4x4, got {tuple(Tb.shape)} and {tuple(Ta.shape)}")
        A = torch.linalg.inv(Ta) @ Tb
        R, t = A[:3, :3], A[:3, 3]
        # log R: the axis-angle vector (theta in [0, pi]), by the skew part away from pi and the symmetric part near it
        c = float(torch.clamp((torch.trace(R) - 1.0) / 2.0, -1.0, 1.0))
        theta = math.acos(c)
        skew = torch.stack([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
        if theta < 1e-6:
            w = 0.5 * skew
        elif math.pi - theta > 1e-4:
            w = (theta / (2.0 * math.sin(theta))) * skew
        else:
            B = (R + torch.eye(3, dtype=torch.float64)) / 2.0
            k = int(torch.argmax(torch.diagonal(B)))
            axis = B[:, k] / torch.sqrt(B[k, k])
            axis = axis * torch.sign(torch.dot(axis, skew)) if float(torch.dot(axis, skew)) != 0.0 else axis
            w = theta * axis
        return MotionBlur(tuple((f * t).tolist()), tuple((f * w).tolist()))

    @property
    def motion(self) -> Tuple[float, ...]:
        """(v, w) as six floats, the order of ``GsbMotionBlurArgs::motion``."""
        return self.linear + self.angular


@dataclass(frozen=True)
class Defocus:
    """The thin lens of a view with depth of field (definition in ``include/gsb200.h``), as host floats: ``aperture`` = a, the
    aperture (entrance pupil) diameter in scene units, and ``focus_distance`` in scene units (``math.inf``: focused at
    infinity).  A point at depth z is blurred to a disk of a f_px |1/focus_distance - 1/z| pixels.  Both values live on the
    normalised image plane, so downsampling, crop and autoscale keep them.

    Two properties of the model: only |a| is observable, and both parameter gradients vanish at a = 0, so refining them needs a
    non-zero start; the focus distance is identifiable only from a view that spans a range of depths (points in front of and
    behind the focal plane blur alike)."""
    aperture: float
    focus_distance: float = math.inf

    def __post_init__(self):
        a, d = float(self.aperture), float(self.focus_distance)
        if not (math.isfinite(a) and a >= 0.0):
            raise ValueError(f"defocus aperture must be finite and >= 0, got {self.aperture}")
        if not (d > 0.0):  # inf allowed, NaN refused
            raise ValueError(f"defocus focus_distance must be > 0 (inf allowed), got {self.focus_distance}")
        object.__setattr__(self, "aperture", a)
        object.__setattr__(self, "focus_distance", d)

    @staticmethod
    def from_lens(focal_length_mm: float, f_number: float, focus_distance: float, units_per_metre: float) -> "Defocus":
        """The thin lens of a photo's EXIF values: the focal length in mm, the f-number N and the focus (subject) distance in
        metres (``math.inf`` for infinity), for a scene ``units_per_metre`` scene units to the metre.  The entrance pupil's
        diameter is f / N."""
        f, n, d, u = float(focal_length_mm), float(f_number), float(focus_distance), float(units_per_metre)
        for name, v in (("focal_length_mm", f), ("f_number", n), ("units_per_metre", u)):
            if not (math.isfinite(v) and v > 0.0):
                raise ValueError(f"{name} must be finite and > 0, got {v}")
        return Defocus((f / 1000.0) / n * u, d * u)

    @property
    def parameters(self) -> Tuple[float, float]:
        """(a, rho) with rho = 1 / focus distance, the order of ``GsbDefocusArgs``."""
        return self.aperture, 1.0 / self.focus_distance


@dataclass
class CameraInfo:
    camera_intrinsics: torch.Tensor  # 3x3 f32 pinhole matrix (device tensor in the reference)
    camera_height: int
    camera_width: int
    camera_id: int
    distortion: Optional[LensDistortion] = None  # extension: None is the reference's pinhole
    rolling_shutter: Optional[RollingShutter] = None  # extension: None is the reference's global shutter
    motion_blur: Optional[MotionBlur] = None  # extension: None is the reference's instantaneous exposure
    defocus: Optional[Defocus] = None  # extension: None is the reference's pinhole, sharp at every depth


@dataclass
class CameraView:
    camera_view_id: int
    T_pointcloud_camera: torch.Tensor  # 4x4 SE(3), camera frame -> pointcloud frame
    camera_id: int
    image_id: int
    timestamp: Optional[int] = None


def orthographic_view(centre: Sequence[float], forward: Sequence[float], up: Sequence[float], width: int, height: int,
                      pixel_size: float, camera_id: int = 0) -> Tuple[torch.Tensor, torch.Tensor, CameraInfo]:
    """(q_pointcloud_camera (1,4) xyzw, t_pointcloud_camera (1,3), CameraInfo) of an orthographic camera at ``centre`` looking
    along ``forward``, with ``up`` toward the top of the image (made orthogonal to ``forward``), ``pixel_size`` scene units per
    pixel.  The orthophoto recipe: a nadir view (``forward`` = -``up`` of the scene, ``up`` any horizontal direction that
    should point to the top of the image) above the scene; where alpha >= 1/2 the surface height is centre . up_scene - depth.
    ``camera_id`` keys the trainer's intrinsics correction: give orthographic views an id of their own when they train
    beside pinhole views, so that refining the pixel size does not move a lens' focal length.  ``ValueError`` for a zero or
    non-finite direction, or ``up`` parallel to ``forward``."""
    from .utils import rotation_matrix_to_quaternion_torch
    c = torch.as_tensor(centre, dtype=torch.float64).reshape(3)
    f = torch.as_tensor(forward, dtype=torch.float64).reshape(3)
    u = torch.as_tensor(up, dtype=torch.float64).reshape(3)
    if not (bool(torch.isfinite(c).all()) and bool(torch.isfinite(f).all()) and bool(torch.isfinite(u).all())):
        raise ValueError("centre, forward and up must be finite")
    if float(f.norm()) == 0.0:
        raise ValueError("forward must not be zero")
    z = f / f.norm()
    down = -(u - torch.dot(u, z) * z)  # the camera's y axis points down the image
    if float(down.norm()) <= 1e-9 * max(float(u.norm()), 1e-300):
        raise ValueError("up must not be zero or parallel to forward")
    y = down / down.norm()
    x = torch.linalg.cross(y, z)
    R = torch.stack([x, y, z], dim=1)  # columns: the camera axes in the scene frame
    q = rotation_matrix_to_quaternion_torch(R[None]).to(torch.float32)
    K = LensDistortion.orthographic_intrinsics(width, height, pixel_size)
    ci = CameraInfo(camera_intrinsics=K, camera_height=int(height), camera_width=int(width), camera_id=int(camera_id),
                    distortion=LensDistortion("orthographic", ()))
    return q.contiguous(), c.to(torch.float32)[None].contiguous(), ci
