"""Drop-in replacement of the reference operator ``GaussianPointCloudRasterisation``.

Same public surface as ``taichi_3d_gaussian_splatting/GaussianPointCloudRasterisation.py:775-1204``
of the reference: ``GaussianPointCloudRasterisation(config, backward_valid_point_hook)`` is an
``nn.Module`` whose ``forward(GaussianPointCloudRasterisationInput)`` returns
``(image (H,W,3) f32, depth (H,W) f32, pixel_valid_point_count (H,W) i32)`` and whose autograd
backward produces dense ``(N,3)`` / ``(N,56)`` gradients, scales them with the fixed factors,
and calls the ``BackwardValidPointHookInput`` side channel -- but every kernel is hand-written
sm_90a CUDA behind the C ABI of ``libgsb200.so`` (``include/gsb200.h``).  PyTorch is used only
for device memory, streams and autograd plumbing.  There is no CPU fallback.

Contract details kept from the reference (SURVEY.md §8(b), §9):
* in-frustum rows of ``point_cloud_features[:, 0:4]`` are normalised IN PLACE each forward
  (GPCR:264-266);
* backward does nothing (all ``None``) unless xyz or features require grad (GPCR:1028);
* the hook runs synchronously inside backward, after gradient scaling (GPCR:1127-1142);
* ``grad_*_factor`` are un-annotated class constants, i.e. not dataclass fields (GPCR:782-786);
* ``camera_width`` / ``camera_height`` must be multiples of 16 (GPCR:1193-1194).
Defined where the reference leaves memory uninitialised: an empty frame (no splat reaches a tile)
renders zeros, and with ``rgb_only=True`` the auxiliary outputs are zeros.
"""
import ctypes
import math
import os
import threading
from dataclasses import dataclass
from typing import Callable, Optional

import torch

from . import _lib
from .Camera import CameraInfo, CameraView  # noqa: F401  (re-exported like the reference module)

BOUNDARY_TILES = 3
TILE_WIDTH = 16
TILE_HEIGHT = 16

_RECORD_FLOATS = 12
_ACCUM_FLOATS = 12


# The projection of a pinhole, OpenCV or fisheye view: the perspective divide, with or without a GsbLensArgs
_PERSPECTIVE = "perspective"

# The lens argument of an equirectangular view: it has no GsbLensArgs and goes through gsb200_forward_equirect /
# gsb200_backward_equirect
_EQUIRECT = "equirectangular"


def _is_equirect(camera_info) -> bool:
    distortion = getattr(camera_info, "distortion", None)
    return distortion is not None and distortion.model == "equirectangular"


# The lens argument of an orthographic view: it has no GsbLensArgs and goes through gsb200_forward_ortho /
# gsb200_backward_ortho
_ORTHO = "orthographic"


def _is_ortho(camera_info) -> bool:
    distortion = getattr(camera_info, "distortion", None)
    return distortion is not None and distortion.model == "orthographic"


# The inputs of the autograd function, in order; an absent optional input is None in its slot
(_XYZ, _FEATURES, _INVALID_MASK, _OBJECT_ID, _Q, _T, _CAMERA_INFO, _SH_BAND, _EXTRA_FEATURES, _INTRINSICS,
 _LENS_COEFFICIENTS, _ROLLING_SHUTTER_MOTION, _FILTER_3D, _EXPOSURE_MOTION, _DEFOCUS_PARAMETERS) = range(15)
_NUM_INPUTS = 15

# The camera-parameter gradient outputs of the backward by input slot: the C argument (output, temp), the gradient's
# shape and the library function that sizes the temp
_CAMERA_GRADS = {
    _INTRINSICS: (_lib.GsbIntrinsicsGradArgs, (3, 3), "gsb200_intrinsics_grad_temp_bytes"),
    _LENS_COEFFICIENTS: (_lib.GsbLensGradArgs, (5,), "gsb200_lens_grad_temp_bytes"),
    _ROLLING_SHUTTER_MOTION: (_lib.GsbRollingShutterGradArgs, (6,), "gsb200_rolling_shutter_grad_temp_bytes"),
    _EXPOSURE_MOTION: (_lib.GsbMotionBlurGradArgs, (6,), "gsb200_motion_blur_grad_temp_bytes"),
    _DEFOCUS_PARAMETERS: (_lib.GsbDefocusGradArgs, (2,), "gsb200_defocus_grad_temp_bytes"),
}


@dataclass
class _Camera:
    """The camera of one call, resolved before any device work from ``camera_info``, the optional tensors and the
    operator's options: the projection, the C arguments of the view's extensions (None where the view has none), and
    the length and device of each camera-parameter tensor passed (lens coefficients, motions, (a, rho)), whose gradient
    goes back sliced to that length on that device."""
    projection: str  # _PERSPECTIVE (pinhole, or the OpenCV / fisheye ``lens``), _EQUIRECT or _ORTHO
    lens: Optional[_lib.GsbLensArgs]
    rolling_shutter: Optional[_lib.GsbRollingShutterArgs]  # its row_time is set by the forward
    motion_blur: Optional[_lib.GsbMotionBlurArgs]
    defocus: Optional[_lib.GsbDefocusArgs]
    filter_3d: Optional[_lib.GsbFilter3dArgs]
    point_filter_3d: Optional[torch.Tensor]  # the array filter_3d points at, kept alive for the backward
    gradient_like: dict  # input slot -> (length, device)
    row_time: Optional[torch.Tensor] = None  # tau_3 of every scene row: written by the forward, read by its backward



def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _ref(s: Optional[ctypes.Structure]):
    """A C struct argument by reference (None stays NULL)."""
    return None if s is None else ctypes.byref(s)


def _f32(t: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    """An incoming gradient as the contiguous float32 tensor the kernels read (None stays None)."""
    if t is None:
        return None
    t = t.contiguous()
    return t if t.dtype == torch.float32 else t.float()


def _require(t: torch.Tensor, name: str, dtype: torch.dtype, shape_tail=None) -> torch.Tensor:
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name} must be a torch.Tensor")
    if not t.is_cuda:
        raise RuntimeError(f"{name} must live on a CUDA device: the rasteriser has no CPU path")
    if t.dtype != dtype:
        raise TypeError(f"{name} must be {dtype}, got {t.dtype}")
    if shape_tail is not None and tuple(t.shape[1:]) != tuple(shape_tail):
        raise ValueError(f"{name} must have shape (*, {', '.join(map(str, shape_tail))}), got {tuple(t.shape)}")
    return t


class _PinnedCounters:
    """Per-device pool of (pinned int64[4] read-back buffer, CUDA event) pairs, one per frame in flight."""
    _free = {}
    _lock = threading.Lock()  # operators of several threads (one per stream) share the pool

    @classmethod
    def acquire(cls, device: torch.device):
        key = device.index if device.index is not None else torch.cuda.current_device()
        with cls._lock:
            pool = cls._free.setdefault(key, [])
            if pool:
                return pool.pop()
        event = torch.cuda.Event()
        event.record()  # materialises the underlying cudaEvent_t so that its handle can cross the C ABI
        return torch.zeros(4, dtype=torch.int64).pin_memory(), event

    @classmethod
    def release(cls, device: torch.device, item) -> None:
        key = device.index if device.index is not None else torch.cuda.current_device()
        with cls._lock:
            cls._free.setdefault(key, []).append(item)


class Frame:
    """Per-call state shared by forward and backward: the workspace blob and typed views into it.

    The views expose the intermediates that the reference keeps as separate saved tensors
    (GPCR:998-1019); tests read them to compare stage by stage against the oracle.
    """

    def __init__(self, ws: torch.Tensor, layout: _lib.GsbWorkspaceLayout, num_points: int,
                 key_capacity: int, height: int, width: int, flags: int):
        self.ws = ws
        self.layout = layout
        self.num_points = num_points
        self.key_capacity = key_capacity
        self.height = height
        self.width = width
        self.flags = flags
        self.num_points_in_camera: Optional[int] = None  # M
        self.num_keys: Optional[int] = None  # K

    def _view(self, offset: int, count: int, dtype: torch.dtype) -> torch.Tensor:
        nbytes = count * torch.empty((), dtype=dtype).element_size()
        return self.ws[offset:offset + nbytes].view(dtype)

    @property
    def counters(self) -> torch.Tensor:
        return self._view(self.layout.counters, 8, torch.int64)

    def _m(self) -> int:
        if self.num_points_in_camera is None:
            raise RuntimeError("frame counters have not been read back yet")
        return self.num_points_in_camera

    @property
    def point_id_in_camera_list(self) -> torch.Tensor:
        return self._view(self.layout.point_id, self.num_points, torch.int32)[:self._m()]

    @property
    def num_overlap_tiles(self) -> torch.Tensor:
        return self._view(self.layout.num_tiles, self.num_points, torch.int32)[:self._m()]

    @property
    def records(self) -> torch.Tensor:
        """(M, 12): u v a b | c rescale opacity depth | r g b radius."""
        return self._view(self.layout.records, self.num_points * _RECORD_FLOATS,
                          torch.float32).view(-1, _RECORD_FLOATS)[:self._m()]

    @property
    def point_in_camera(self) -> torch.Tensor:
        return self._view(self.layout.point_in_camera, self.num_points * 3, torch.float32).view(-1, 3)[:self._m()]

    @property
    def point_uv(self) -> torch.Tensor:
        return self.records[:, 0:2]

    @property
    def point_uv_conic_and_rescale(self) -> torch.Tensor:
        r = self.records
        return torch.stack([r[:, 2], r[:, 3], r[:, 4], r[:, 5]], dim=-1)

    @property
    def point_alpha_after_activation(self) -> torch.Tensor:
        return self.records[:, 6]

    @property
    def point_color(self) -> torch.Tensor:
        return self.records[:, 8:11]

    @property
    def point_radii(self) -> torch.Tensor:
        return self.records[:, 11]

    @property
    def sorted_keys(self) -> torch.Tensor:
        """Sorted packed keys (tile << depth_bits | depth), int64 regardless of the device key width."""
        off = self.layout.keys_b  # the sort always ends in b
        n = min(self.num_keys, self.key_capacity)
        if self.layout.key_bytes == 4:
            return self._view(off, self.layout.key_capacity_padded, torch.int32)[:n].to(torch.int64) & 0xFFFFFFFF
        return self._view(off, self.layout.key_capacity_padded, torch.int64)[:n]

    @property
    def point_offset_with_sort_key(self) -> torch.Tensor:
        off = self.layout.vals_b
        n = min(self.num_keys, self.key_capacity)
        return self._view(off, self.layout.key_capacity_padded, torch.int32)[:n]

    @property
    def tile_points_start(self) -> torch.Tensor:
        T = (self.height // TILE_HEIGHT) * (self.width // TILE_WIDTH)
        return self._view(self.layout.tile_start, T, torch.int32)

    @property
    def tile_points_end(self) -> torch.Tensor:
        T = (self.height // TILE_HEIGHT) * (self.width // TILE_WIDTH)
        return self._view(self.layout.tile_end, T, torch.int32)


class GaussianPointCloudRasterisation(torch.nn.Module):
    @dataclass
    class GaussianPointCloudRasterisationConfig:
        # reference: GPCR:776-786 (a dataclass_wizard YAMLWizard there; plain dataclass here)
        near_plane: float = 0.8
        far_plane: float = 1000.
        depth_to_sort_key_scale: float = 100.
        rgb_only: bool = False
        # un-annotated on purpose: class constants, not dataclass fields (GPCR:782-786)
        grad_color_factor = 5.
        grad_high_order_color_factor = 1.
        grad_s_factor = 0.5
        grad_q_factor = 1.
        grad_alpha_factor = 20.

    @dataclass
    class GaussianPointCloudRasterisationInput:
        # reference: GPCR:788-804
        point_cloud: torch.Tensor  # Nx3
        point_cloud_features: torch.Tensor  # Nx56
        point_object_id: torch.Tensor  # N, int32
        point_invalid_mask: torch.Tensor  # N, int8
        camera_info: CameraInfo
        q_pointcloud_camera: torch.Tensor  # Kx4 (x, y, z, w), camera -> pointcloud
        t_pointcloud_camera: torch.Tensor  # Kx3
        color_max_sh_band: int = 2

    @dataclass
    class BackwardValidPointHookInput:
        # reference: GPCR:806-817
        point_id_in_camera_list: torch.Tensor  # M
        grad_point_in_camera: torch.Tensor  # Mx3
        grad_pointfeatures_in_camera: torch.Tensor  # Mx56
        grad_viewspace: torch.Tensor  # Mx2
        magnitude_grad_viewspace: torch.Tensor  # M
        magnitude_grad_viewspace_on_image: torch.Tensor  # HxWx2
        num_overlap_tiles: torch.Tensor  # M
        num_affected_pixels: torch.Tensor  # M
        point_depth: torch.Tensor  # M
        point_uv_in_camera: torch.Tensor  # Mx2

    def __init__(
        self,
        config: "GaussianPointCloudRasterisation.GaussianPointCloudRasterisationConfig",
        backward_valid_point_hook: Optional[Callable[["GaussianPointCloudRasterisation.BackwardValidPointHookInput"], None]] = None,
        *,
        exact_exp: bool = False,
        force_key64: bool = False,
        initial_key_capacity: Optional[int] = None,
        keep_all_tile_pairs: bool = False,
        backward_impl: Optional[str] = None,
        skip_unused_hook_statistics: Optional[bool] = None,
        gradient_exchange=None,
        differentiable_depth: bool = False,
        differentiable_alpha: bool = False,
        differentiable_pose: bool = False,
        differentiable_intrinsics: bool = False,
        differentiable_distortion: bool = False,
        differentiable_rolling_shutter: bool = False,
        differentiable_motion_blur: bool = False,
        differentiable_defocus: bool = False,
        camera_gradients_through_lens: bool = False,
    ):
        """``exact_exp``: blend kernels use ``expf`` instead of ``ex2.approx`` (parity debugging).
        ``force_key64``: sort the reference's 64-bit ``tile << 32 | depth`` keys even when the live
        bits fit 32.  ``initial_key_capacity``: first guess for the number of (tile, splat) pairs;
        the buffers grow automatically when a frame needs more.  ``keep_all_tile_pairs``: emit a sort key for
        every tile of the reference's 3-sigma square instead of only the tiles the splat can actually reach with
        alpha >= 1/255 (same outputs, ~1.5x more keys; used by tests that compare the sorted list itself).
        ``backward_impl``: ``"transposed"`` (default; ``csrc/blend_bwd_transposed.cu``: splat-per-lane accumulation after a
        shared-memory transposition) or ``"butterfly"`` (``csrc/blend_bwd.cu``: warp butterfly per (warp, splat), slower;
        kept as the second implementation the parity tests cross-check).  Constructor argument only:
        no environment variable can switch the kernel of a production run.  With no backward hook installed the transposed
        kernel does not compute the statistics only a hook reads (the reference's ``need_extra_info = False``, GPCR:521).
        ``skip_unused_hook_statistics``: the same switch for the butterfly kernel (opt-in; ``None`` reads
        ``GSB200_SKIP_HOOK_STATS``).
        ``gradient_exchange``: a ``parallel.ViewParallelExchange`` (view-parallel training, one process per GPU): backward
        then returns the gradients SUMMED over the ranks' views -- the per-point kernel writes compact rows, the ranks
        exchange 14 instead of 59 floats per Gaussian and ``gsb200_expand_view_gradients`` rebuilds the dense sum.  A
        backward hook still sees this rank's own view (``grad_pointfeatures_in_camera`` is ``None`` in this mode: the
        per-view dense feature gradients are never formed).
        ``differentiable_depth``: make the returned depth map differentiable (an extension: the reference's depth output is
        not, and by default neither is ours).  A loss on depth then trains xyz, q, s and the opacity through the blend
        weights, and xyz also through each splat's camera-space depth (``gsb200_backward_with_depth``); a loss on depth
        alone works too.  The hook sees the sum of both losses' shares in ``grad_point_in_camera``, ``grad_viewspace``
        and the magnitudes, exactly as it sees the image loss's share.  Needs the transposed backward and the auxiliary
        outputs: ``ValueError`` with ``backward_impl="butterfly"`` or ``config.rgb_only``.
        ``differentiable_alpha``: ``forward`` also returns the per-pixel accumulated alpha S = 1 - prod (1 - alpha), (H, W)
        float32, as a fourth output, differentiable (``gsb200_backward_aux``): a mask loss on S, or an image composited
        on a background as ``image + (1 - S)[..., None] * bg``, trains xyz, q, s and the opacity through the blend weights;
        a loss on S alone works too.  Combines with ``differentiable_depth``.  The hook sees the alpha loss's share as it
        sees the image loss's share.  Same requirements as ``differentiable_depth``: ``ValueError`` with
        ``backward_impl="butterfly"`` or ``config.rgb_only``.
        ``differentiable_pose``: ``backward`` also returns dL/d ``q_pointcloud_camera`` (K, 4) and dL/d
        ``t_pointcloud_camera`` (K, 3) for whichever of them requires grad (an extension: the reference differentiates the
        scene only) -- to refine noisy training poses, relocalise a camera against a trained scene, or track rigid objects
        (one pose per ``point_object_id``).  The gradient is exact through the pose map of the forward (q is conjugated,
        normalised for the translation and taken as given for the rotation), with the point gradients' conventions (J and
        the SH view direction detached), and includes every loss term the backward takes (image, depth, alpha, features);
        no gradient factor is applied (``gsb200_backward_pose``).  With a frozen scene (only q / t require grad) the backward
        still runs.  At most 64 objects.  An image-only loss works with either backward kernel.  Off, a pose that requires
        grad gets ``None``.  ``ValueError`` with ``config.rgb_only`` or a ``gradient_exchange``.
        ``differentiable_intrinsics``: ``camera_info.camera_intrinsics`` becomes an input of the autograd graph, and
        ``backward`` returns its (3, 3) gradient when it requires grad (an extension: the reference differentiates the scene
        only) -- to calibrate focal length and principal point, alone or together with the poses, also against a frozen
        scene and also for a K built by torch ops from learnable parameters.  The gradient is exact through the projection
        uv = (K pc)[:2] / z (all six entries of rows 0 and 1) and through fx, fy inside J, with the conventions of the point
        and pose gradients (J's dependence on pc, the rescale factor, tile membership and the SH view direction detached);
        row 2 gets 0, and no gradient factor is applied (``gsb200_backward_calib``).  It includes every loss term the
        backward takes (image, depth, alpha, features).  With ``differentiable_pose`` both come from one pass of the
        per-point kernel.  An image-only loss works with either backward kernel.  Off, K gets no gradient.  ``ValueError``
        with ``config.rgb_only`` or a ``gradient_exchange``.
        ``differentiable_distortion``: ``forward`` takes ``lens_coefficients``, the values of ``camera_info.distortion``'s
        coefficients as an input of the autograd graph, and ``backward`` returns their gradient -- to refine a lens that is
        roughly known (a pinhole or one-coefficient COLMAP model of a lens that distorts, a generic fisheye profile).  The
        gradient is exact through the position and through D inside J, with the conventions of the point, pose and
        intrinsics gradients (D at the detached point, rescale, tile membership and the SH view direction detached, the
        r_max cut not differentiated); it includes every loss term the backward takes (image, depth, alpha, features), and no
        gradient factor is applied (``gsb200_backward_lens_grad``).  An image-only loss works with either backward kernel.
        ``ValueError`` with ``config.rgb_only`` or a ``gradient_exchange``; like every lens, not with
        ``differentiable_pose`` or ``differentiable_intrinsics`` unless ``camera_gradients_through_lens`` is set.
        ``differentiable_rolling_shutter``: ``forward`` takes ``rolling_shutter_motion``, the values of
        ``camera_info.rolling_shutter``'s motion (v, w) as an input of the autograd graph, and ``backward`` returns their
        gradient -- to refine the camera motion of a phone, action-camera or drone view whose velocity is roughly known or
        unknown.  The row time is detached; the gradient flows through pc(tau) and Rd(tau) W (``gsb200_backward_rolling_shutter``,
        definition in ``include/gsb200.h``) and includes every loss term the backward takes (image, depth, alpha, features).
        An image-only loss works with either backward kernel.  ``ValueError`` with ``config.rgb_only`` or a
        ``gradient_exchange``.
        ``differentiable_motion_blur``: ``forward`` takes ``exposure_motion``, the values of ``camera_info.motion_blur``'s
        motion (v, w) as an input of the autograd graph, and ``backward`` returns their gradient -- to refine the exposure
        motion of a blurred view from a non-zero start (the gradient vanishes at zero motion).  d is detached; the gradient
        flows through B = d d^T / 12 and the compensation c_b (``gsb200_backward_motion_blur``, definition in
        ``include/gsb200.h``) and includes every loss term the backward takes (image, depth, alpha, features).  An image-only
        loss works with either backward kernel.  ``ValueError`` with ``config.rgb_only`` or a ``gradient_exchange``.
        ``differentiable_defocus``: ``forward`` takes ``defocus_parameters``, the values (a, rho) of ``camera_info.defocus``
        as an input of the autograd graph, and ``backward`` returns their gradient -- to refine the aperture and focus
        distance of a defocused view from a non-zero aperture (both gradients vanish at a = 0).  beta is detached with respect
        to the point; the gradient flows through B_d = beta M M^T and the compensation c_b (``gsb200_backward_defocus``,
        definition in ``include/gsb200.h``) and includes every loss term the backward takes (image, depth, alpha, features).
        ``ValueError`` with ``config.rgb_only`` or a ``gradient_exchange``.
        ``camera_gradients_through_lens`` (opt-in): ``differentiable_pose`` and ``differentiable_intrinsics`` also
        differentiate an OpenCV or fisheye view, alone, together and with ``differentiable_distortion`` -- photometric
        self-calibration of the poses, K and the lens of ordinary COLMAP output.  All three camera gradients come from one
        pass of the per-point kernel (``gsb200_backward_lens_calib``; the model is in ``include/gsb200.h``): d uv / d pc =
        K[:2,:2] D P, J = diag(fx, fy) D P inside Sigma', and dL/dK[r] through (xd, yd, 1), with the conventions of the
        pinhole gradients (J and D at the detached point, the r_max cut not differentiated).  Without it a lens keeps refusing
        the two options (``ValueError``), as before.  It changes nothing for a pinhole or orthographic view.  Camera
        gradients stay refused with a rolling shutter, motion blur, defocus, an equirectangular panorama, ``point_filter_3d``
        and a ``gradient_exchange``; the depth, alpha and feature terms keep needing the transposed backward kernel."""
        super().__init__()
        for name, on in (("differentiable_depth", differentiable_depth), ("differentiable_alpha", differentiable_alpha)):
            if on and backward_impl == "butterfly":
                raise ValueError(f"{name} needs backward_impl='transposed': the butterfly kernel implements only the "
                                 "image gradient")
            if on and config.rgb_only:
                raise ValueError(f"{name} needs the auxiliary outputs: config.rgb_only=True renders none")
        self.differentiable_depth = bool(differentiable_depth)
        self.differentiable_alpha = bool(differentiable_alpha)
        for name, on in (("differentiable_pose", differentiable_pose), ("differentiable_intrinsics", differentiable_intrinsics),
                         ("differentiable_distortion", differentiable_distortion),
                         ("differentiable_rolling_shutter", differentiable_rolling_shutter),
                         ("differentiable_motion_blur", differentiable_motion_blur),
                         ("differentiable_defocus", differentiable_defocus)):
            if on and config.rgb_only:
                raise ValueError(f"{name} needs the auxiliary outputs: config.rgb_only=True renders none")
            if on and gradient_exchange is not None:
                raise ValueError(f"{name} is not supported with a gradient_exchange (view-parallel training)")
        self.differentiable_pose = bool(differentiable_pose)
        self.differentiable_intrinsics = bool(differentiable_intrinsics)
        self.differentiable_distortion = bool(differentiable_distortion)
        self.differentiable_rolling_shutter = bool(differentiable_rolling_shutter)
        self.differentiable_motion_blur = bool(differentiable_motion_blur)
        self.differentiable_defocus = bool(differentiable_defocus)
        self.camera_gradients_through_lens = bool(camera_gradients_through_lens)
        self.config = config
        self.backward_valid_point_hook = backward_valid_point_hook
        self._flags = (_lib.GSB_FLAG_EXACT_EXP if exact_exp else 0) | (_lib.GSB_FLAG_FORCE_KEY64 if force_key64 else 0) | \
            (_lib.GSB_FLAG_KEEP_ALL_TILE_PAIRS if keep_all_tile_pairs else 0)
        backward_impl = backward_impl or "transposed"
        if backward_impl not in ("butterfly", "transposed"):
            raise ValueError(f"backward_impl must be 'butterfly' or 'transposed', got {backward_impl!r}")
        self.backward_impl = backward_impl
        if skip_unused_hook_statistics is None:
            skip_unused_hook_statistics = os.environ.get("GSB200_SKIP_HOOK_STATS", "0") not in ("", "0")
        self.skip_unused_hook_statistics = bool(skip_unused_hook_statistics)
        self.gradient_exchange = gradient_exchange
        self._key_capacity = int(initial_key_capacity) if initial_key_capacity else 0
        self.last_frame: Optional[Frame] = None
        self.last_gradient_buffer: Optional[torch.Tensor] = None  # flat storage behind the latest backward's grads
        self._layout_cache = {}
        _lib.load()  # fail loudly at construction time if the CUDA library is missing
        outer = self

        class _module_function(torch.autograd.Function):

            @staticmethod
            def forward(ctx, pointcloud, pointcloud_features, point_invalid_mask, point_object_id,
                        q_pointcloud_camera, t_pointcloud_camera, camera_info, color_max_sh_band, extra_features,
                        camera_intrinsics, lens_coefficients, rolling_shutter_motion, point_filter_3d, exposure_motion,
                        defocus_parameters):
                # camera_intrinsics (differentiable_intrinsics): camera_info.camera_intrinsics itself, passed again only so
                # that autograd tracks it; lens_coefficients (differentiable_distortion): the coefficients rendered;
                # rolling_shutter_motion (differentiable_rolling_shutter): the motion rendered; point_filter_3d: the 3D
                # smoothing filter (never differentiated); exposure_motion (differentiable_motion_blur): the exposure motion
                # rendered; defocus_parameters (differentiable_defocus): the (a, rho) rendered
                camera = outer._resolve_camera(camera_info, pointcloud, extra_features, lens_coefficients,
                                               rolling_shutter_motion, point_filter_3d, exposure_motion, defocus_parameters)
                outs, frame, K = outer._run_forward(camera, pointcloud, pointcloud_features, point_invalid_mask,
                                                    point_object_id, q_pointcloud_camera, t_pointcloud_camera, camera_info,
                                                    extra_features)
                image, depth, acc_alpha, last_effective, valid_count = outs[:5]
                ctx.save_for_backward(pointcloud, pointcloud_features, point_object_id,
                                      q_pointcloud_camera if outer.differentiable_pose else None, t_pointcloud_camera, K,
                                      acc_alpha, last_effective, frame.ws, depth if outer.differentiable_depth else None,
                                      extra_features)
                ctx.frame = frame
                ctx.camera = camera
                ctx.num_objects = q_pointcloud_camera.shape[0]
                ctx.color_max_sh_band = color_max_sh_band
                if outer.differentiable_depth:
                    ctx.mark_non_differentiable(valid_count)
                else:
                    ctx.mark_non_differentiable(depth, valid_count)
                if outer.differentiable_depth or outer.differentiable_alpha or extra_features is not None:
                    ctx.set_materialize_grads(False)  # None tells an unused output from a zero gradient
                result = (image, depth, valid_count) + ((acc_alpha,) if outer.differentiable_alpha else ())
                if extra_features is not None:
                    result = result + (outs[5],)
                return result

            @staticmethod
            def backward(ctx, grad_rasterized_image, grad_rasterized_depth, grad_pixel_valid_point_count, *grad_extra):
                # grad_extra: dL/d pixel_accumulated_alpha (differentiable_alpha), then dL/d the feature map (extra features)
                grad_pixel_accumulated_alpha = grad_extra[0] if outer.differentiable_alpha else None
                grad_feature_map = grad_extra[-1] if len(grad_extra) > int(outer.differentiable_alpha) else None
                needs = ctx.needs_input_grad
                pose = outer.differentiable_pose and (needs[_Q] or needs[_T])
                camera_grads = [slot for slot in _CAMERA_GRADS if needs[slot]]
                result = [None] * _NUM_INPUTS
                # GPCR:1028; with extra features or camera-parameter gradients the backward also runs for them alone
                # (frozen scene)
                if needs[_XYZ] or needs[_FEATURES] or needs[_EXTRA_FEATURES] or pose or camera_grads:
                    if outer.config.rgb_only:
                        # the reference leaves accumulated alpha / last-effective offsets uninitialised in
                        # this mode (GPCR:478-484), so its backward is undefined; refuse instead
                        raise RuntimeError("rgb_only=True is an inference-only mode: backward needs the "
                                           "auxiliary per-pixel outputs")
                    if grad_rasterized_image is None:  # a loss on the depth map or the accumulated alpha alone
                        frame = ctx.frame
                        grad_rasterized_image = torch.zeros((frame.height, frame.width, 3), dtype=torch.float32,
                                                            device=frame.ws.device)
                    grads = outer._run_backward(ctx, grad_rasterized_image, grad_rasterized_depth,
                                                grad_pixel_accumulated_alpha, grad_feature_map, pose, camera_grads)
                    for slot, grad in grads.items():
                        if needs[slot]:
                            result[slot] = grad
                return tuple(result)

        self._module_function = _module_function

    # ------------------------------------------------------------------ forward plumbing
    def _default_key_capacity(self, num_points: int) -> int:
        return max(1 << 20, 8 * num_points)

    def _layout(self, N, n_obj, key_capacity, H, W):
        key = (N, n_obj, key_capacity, H, W, self.config.far_plane, self.config.depth_to_sort_key_scale, self._flags)
        cached = self._layout_cache.get(key)
        if cached is None:
            if len(self._layout_cache) > 64:
                self._layout_cache.clear()
            cached = _lib.workspace_layout(N, n_obj, key_capacity, H, W, self.config.far_plane,
                                           self.config.depth_to_sort_key_scale, self._flags)
            self._layout_cache[key] = cached
        return cached

    def _check_extra_features(self, extra_features, pointcloud):
        """The ``point_extra_features`` argument of ``forward``: (N, C) float32, contiguous, on the scene's device, 1 <= C <= 16,
        and an operator that can differentiate it."""
        if self.backward_impl == "butterfly":
            raise ValueError("point_extra_features needs backward_impl='transposed': the butterfly kernel implements only the "
                             "image gradient")
        if self.config.rgb_only:
            raise ValueError("point_extra_features needs the full forward: config.rgb_only=True renders only the image")
        if self.gradient_exchange is not None:
            raise ValueError("point_extra_features is not supported with a gradient_exchange (view-parallel training)")
        if not isinstance(extra_features, torch.Tensor):
            raise ValueError("point_extra_features must be a torch.Tensor")
        N = pointcloud.shape[0]
        if extra_features.dim() != 2 or extra_features.shape[0] != N or not 1 <= extra_features.shape[1] <= 16:
            raise ValueError(f"point_extra_features must be (N, C) with N = {N} and 1 <= C <= 16, got "
                             f"{tuple(extra_features.shape)}")
        if extra_features.dtype != torch.float32:
            raise ValueError(f"point_extra_features must be float32, got {extra_features.dtype}")
        if extra_features.device != pointcloud.device:
            raise ValueError(f"point_extra_features must be on {pointcloud.device}, got {extra_features.device}")
        if not extra_features.is_contiguous():
            raise ValueError("point_extra_features must be contiguous")

    def _check_filter_3d(self, point_filter_3d, pointcloud):
        """The ``point_filter_3d`` argument of ``forward``: (N,) float32, contiguous, on the scene's device, and an operator
        without camera-parameter gradients or a gradient exchange."""
        for name, on in (("differentiable_pose", self.differentiable_pose),
                         ("differentiable_intrinsics", self.differentiable_intrinsics),
                         ("differentiable_distortion", self.differentiable_distortion),
                         ("differentiable_rolling_shutter", self.differentiable_rolling_shutter),
                         ("a gradient_exchange", self.gradient_exchange is not None)):
            if on:
                raise ValueError(f"point_filter_3d is not supported with {name}")
        if not isinstance(point_filter_3d, torch.Tensor):
            raise ValueError("point_filter_3d must be a torch.Tensor")
        N = pointcloud.shape[0]
        if tuple(point_filter_3d.shape) != (N,):
            raise ValueError(f"point_filter_3d must have shape ({N},), got {tuple(point_filter_3d.shape)}")
        if point_filter_3d.dtype != torch.float32:
            raise ValueError(f"point_filter_3d must be float32, got {point_filter_3d.dtype}")
        if point_filter_3d.device != pointcloud.device:
            raise ValueError(f"point_filter_3d must be on {pointcloud.device}, got {point_filter_3d.device}")
        if not point_filter_3d.is_contiguous():
            raise ValueError("point_filter_3d must be contiguous")

    def _resolve_camera(self, camera_info, pointcloud, extra_features=None, lens_coefficients=None,
                        rolling_shutter_motion=None, point_filter_3d=None, exposure_motion=None,
                        defocus_parameters=None) -> _Camera:
        """The camera of a call (``_Camera``), after every argument check that needs no device: each refusal of what the
        view does not combine with is raised here, before any CUDA call."""
        if _is_equirect(camera_info):
            self._check_equirect(camera_info, lens_coefficients, rolling_shutter_motion, point_filter_3d, exposure_motion,
                                 defocus_parameters)
        if _is_ortho(camera_info):
            self._check_ortho(camera_info, lens_coefficients, rolling_shutter_motion, exposure_motion, defocus_parameters)
        assert camera_info.camera_width % TILE_WIDTH == 0
        assert camera_info.camera_height % TILE_HEIGHT == 0
        # Which refusal wins where several apply: defocus, motion blur, the filter and each camera-parameter tensor are
        # checked before the feature channels, a lens or rolling shutter that comes with camera_info alone after them.
        defocus = self._defocus_args(camera_info, defocus_parameters, rolling_shutter_motion, point_filter_3d, exposure_motion)
        blur = self._motion_blur_args(camera_info, exposure_motion, rolling_shutter_motion, point_filter_3d)
        if point_filter_3d is not None:
            for name, value in (("lens_coefficients", lens_coefficients), ("rolling_shutter_motion", rolling_shutter_motion)):
                if value is not None:
                    raise ValueError(f"point_filter_3d is not supported with {name} (no camera-parameter gradient with the "
                                     "filter)")
            self._check_filter_3d(point_filter_3d, pointcloud)
        if rolling_shutter_motion is not None:
            rs = self._rolling_shutter_args(camera_info, rolling_shutter_motion)
        if lens_coefficients is not None:
            lens = self._lens_args(camera_info, lens_coefficients)
        if extra_features is not None:
            self._check_extra_features(extra_features, pointcloud)
        if lens_coefficients is None:
            lens = self._lens_args(camera_info)
        if rolling_shutter_motion is None:
            rs = self._rolling_shutter_args(camera_info)
        projection = lens if lens is _EQUIRECT or lens is _ORTHO else _PERSPECTIVE
        gradient_like = {slot: (t.shape[0], t.device) for slot, t in (
            (_LENS_COEFFICIENTS, lens_coefficients), (_ROLLING_SHUTTER_MOTION, rolling_shutter_motion),
            (_EXPOSURE_MOTION, exposure_motion), (_DEFOCUS_PARAMETERS, defocus_parameters)) if t is not None}
        return _Camera(projection=projection, lens=lens if projection is _PERSPECTIVE else None, rolling_shutter=rs,
                       motion_blur=blur, defocus=defocus,
                       filter_3d=None if point_filter_3d is None else _lib.GsbFilter3dArgs(filter3d=_ptr(point_filter_3d)),
                       point_filter_3d=point_filter_3d, gradient_like=gradient_like)

    def _run_forward(self, camera: _Camera, pointcloud, pointcloud_features, point_invalid_mask, point_object_id,
                     q_pointcloud_camera, t_pointcloud_camera, camera_info, extra_features=None):
        cfg = self.config
        lib = _lib.load()
        _require(pointcloud, "point_cloud", torch.float32, (3,))
        _require(pointcloud_features, "point_cloud_features", torch.float32, (56,))
        _require(point_invalid_mask, "point_invalid_mask", torch.int8)
        _require(point_object_id, "point_object_id", torch.int32)
        _require(q_pointcloud_camera, "q_pointcloud_camera", torch.float32, (4,))
        _require(t_pointcloud_camera, "t_pointcloud_camera", torch.float32, (3,))
        K = camera_info.camera_intrinsics
        _require(K, "camera_info.camera_intrinsics", torch.float32)
        for name, t in (("point_cloud", pointcloud), ("point_cloud_features", pointcloud_features),
                        ("point_invalid_mask", point_invalid_mask), ("point_object_id", point_object_id)):
            if not t.is_contiguous():  # Taichi rejects non-contiguous ndarrays as well
                raise ValueError(f"{name} must be contiguous")
        q_pc = q_pointcloud_camera.contiguous()
        t_pc = t_pointcloud_camera.contiguous()
        K = K.contiguous()
        device = pointcloud.device
        N = pointcloud.shape[0]
        n_obj = q_pc.shape[0]
        H, W = int(camera_info.camera_height), int(camera_info.camera_width)
        if self._key_capacity <= 0:
            self._key_capacity = self._default_key_capacity(N)

        with torch.cuda.device(device):
            stream = torch.cuda.current_stream(device)
            image = torch.empty((H, W, 3), dtype=torch.float32, device=device)
            if cfg.rgb_only:
                depth = torch.zeros((H, W), dtype=torch.float32, device=device)
                acc_alpha = torch.zeros((H, W), dtype=torch.float32, device=device)
                last_effective = torch.zeros((H, W), dtype=torch.int32, device=device)
                valid_count = torch.zeros((H, W), dtype=torch.int32, device=device)
            else:
                depth = torch.empty((H, W), dtype=torch.float32, device=device)
                acc_alpha = torch.empty((H, W), dtype=torch.float32, device=device)
                last_effective = torch.empty((H, W), dtype=torch.int32, device=device)
                valid_count = torch.empty((H, W), dtype=torch.int32, device=device)
            feature_map = ext = None
            if extra_features is not None:
                C = extra_features.shape[1]
                feature_map = torch.empty((H, W, C), dtype=torch.float32, device=device)
                ext = _lib.GsbExtraFeatureArgs(channels=C, features=_ptr(extra_features), rasterized=_ptr(feature_map))
            if camera.rolling_shutter is not None:  # read back by the backward of this frame
                camera.row_time = torch.empty((max(N, 1),), dtype=torch.float32, device=device)
                camera.rolling_shutter.row_time = _ptr(camera.row_time)
            if camera.projection is _EQUIRECT:
                entry, camera_args = "gsb200_forward_equirect", (ext,)
            elif camera.projection is _ORTHO:
                entry, camera_args = "gsb200_forward_ortho", (ext, camera.filter_3d)
            elif camera.motion_blur is not None or camera.defocus is not None:
                entry, camera_args = "gsb200_forward_defocus", (ext, camera.lens, camera.rolling_shutter, camera.motion_blur,
                                                                camera.defocus)
            else:
                entry, camera_args = "gsb200_forward_filter3d", (ext, camera.lens, camera.rolling_shutter, camera.filter_3d)
            readback = _PinnedCounters.acquire(device)
            pinned, event = readback
            retry_flag = 0
            try:
                while True:
                    key_capacity = self._key_capacity
                    layout = self._layout(N, n_obj, key_capacity, H, W)
                    ws = torch.empty((layout.total_bytes,), dtype=torch.uint8, device=device)
                    args = _lib.GsbForwardArgs(
                        num_points=N, pointcloud=_ptr(pointcloud), pointcloud_features=_ptr(pointcloud_features),
                        point_invalid_mask=_ptr(point_invalid_mask), point_object_id=_ptr(point_object_id),
                        num_objects=n_obj, q_pointcloud_camera=_ptr(q_pc), t_pointcloud_camera=_ptr(t_pc),
                        camera_intrinsics=_ptr(K), camera_height=H, camera_width=W,
                        near_plane=cfg.near_plane, far_plane=cfg.far_plane,
                        depth_to_sort_key_scale=cfg.depth_to_sort_key_scale, rgb_only=1 if cfg.rgb_only else 0,
                        flags=self._flags | retry_flag, workspace=_ptr(ws), workspace_bytes=layout.total_bytes,
                        key_capacity=key_capacity, rasterized_image=_ptr(image), rasterized_depth=_ptr(depth),
                        pixel_accumulated_alpha=_ptr(acc_alpha),
                        pixel_offset_of_last_effective_point=_ptr(last_effective),
                        pixel_valid_point_count=_ptr(valid_count), stream=stream.cuda_stream,
                        host_counters=pinned.data_ptr(), host_counters_event=event.cuda_event)
                    # The whole frame is enqueued by this one call; the library copies {M, K, overflow} to pinned
                    # host memory right after the per-point stage and records `event` behind that copy.
                    _lib.check(getattr(lib, entry)(ctypes.byref(args), *map(_ref, camera_args)), entry)
                    frame = Frame(ws, layout, N, key_capacity, H, W, self._flags)
                    # ONE host wait per frame (the reference syncs twice, GPCR:864 and GPCR:916-931), and it ends
                    # when the first kernel is done: sort + blend are still in flight when we return.
                    event.synchronize()
                    frame.num_points_in_camera = int(pinned[0])
                    frame.num_keys = int(pinned[1])
                    if int(pinned[2]) == 0:
                        break
                    # more (tile, splat) pairs than capacity: grow and redo the frame.  The first pass already
                    # normalised the quaternions in place; the re-run must not normalise them a second time.
                    self._key_capacity = int(frame.num_keys * 1.25) + 4096
                    retry_flag = _lib.GSB_FLAG_Q_ALREADY_NORMALISED
            finally:  # also when the library call raises: the pooled pair goes back
                _PinnedCounters.release(device, readback)
        self.last_frame = frame
        outs = (image, depth, acc_alpha, last_effective, valid_count) + ((feature_map,) if feature_map is not None else ())
        return outs, frame, K

    def _lens_args(self, camera_info, lens_coefficients=None) -> Optional[_lib.GsbLensArgs]:
        """The C lens argument of ``camera_info.distortion`` (None: the pinhole kernels), after the checks of the options
        a lens does not combine with; with ``lens_coefficients`` (``differentiable_distortion``) its values replace the
        record's coefficients (read on the host: free for a CPU tensor, one blocking 20-byte copy for a device tensor)."""
        distortion = getattr(camera_info, "distortion", None)
        if lens_coefficients is not None:
            if not self.differentiable_distortion:
                raise ValueError("lens_coefficients needs differentiable_distortion=True")
            if distortion is None:
                raise ValueError("lens_coefficients was given for a camera with no lens (camera_info.distortion is None)")
        if distortion is None:
            return None
        if distortion.model == "equirectangular":
            self._check_equirect(camera_info, lens_coefficients)
            return _EQUIRECT
        if distortion.model == "orthographic":
            self._check_ortho(camera_info, lens_coefficients)
            return _ORTHO
        through = self.camera_gradients_through_lens
        for name, on in (("differentiable_pose", self.differentiable_pose and not through),
                         ("differentiable_intrinsics", self.differentiable_intrinsics and not through),
                         ("a gradient_exchange", self.gradient_exchange is not None)):
            if on:
                hint = "" if name.startswith("a ") else " (camera_gradients_through_lens=True differentiates through it)"
                raise ValueError(f"a camera with lens distortion is not supported with {name}{hint}")
        if lens_coefficients is None:
            return _lib.lens_args(distortion)
        n = len(distortion.coefficients)
        if not isinstance(lens_coefficients, torch.Tensor):
            raise ValueError("lens_coefficients must be a torch.Tensor")
        if tuple(lens_coefficients.shape) != (n,):
            raise ValueError(f"lens_coefficients must have shape ({n},) for the {distortion.model} lens, got "
                             f"{tuple(lens_coefficients.shape)}")
        if lens_coefficients.dtype != torch.float32:
            raise ValueError(f"lens_coefficients must be float32, got {lens_coefficients.dtype}")
        values = lens_coefficients.detach().cpu().tolist()
        return _lib.lens_args(type(distortion)(distortion.model, values))

    def _check_equirect(self, camera_info, lens_coefficients=None, rolling_shutter_motion=None, point_filter_3d=None,
                        exposure_motion=None, defocus_parameters=None) -> None:
        """``ValueError`` for what an equirectangular view does not combine with (include/gsb200.h): camera-parameter
        gradients, the other camera extensions, the 3D filter, the view-parallel exchange and the butterfly backward."""
        for name, on in (("differentiable_pose", self.differentiable_pose),
                         ("differentiable_intrinsics", self.differentiable_intrinsics),
                         ("differentiable_distortion", self.differentiable_distortion),
                         ("differentiable_rolling_shutter", self.differentiable_rolling_shutter),
                         ("differentiable_motion_blur", self.differentiable_motion_blur),
                         ("differentiable_defocus", self.differentiable_defocus),
                         ("a gradient_exchange", self.gradient_exchange is not None),
                         ("backward_impl='butterfly'", self.backward_impl == "butterfly"),
                         ("a rolling shutter (camera_info.rolling_shutter)", getattr(camera_info, "rolling_shutter", None) is not None),
                         ("motion blur (camera_info.motion_blur)", getattr(camera_info, "motion_blur", None) is not None),
                         ("defocus (camera_info.defocus)", getattr(camera_info, "defocus", None) is not None),
                         ("lens_coefficients", lens_coefficients is not None),
                         ("rolling_shutter_motion", rolling_shutter_motion is not None),
                         ("point_filter_3d", point_filter_3d is not None),
                         ("exposure_motion", exposure_motion is not None),
                         ("defocus_parameters", defocus_parameters is not None)):
            if on:
                raise ValueError(f"an equirectangular camera is not supported with {name}")
        if int(camera_info.camera_width) % TILE_WIDTH != 0:
            raise ValueError(f"an equirectangular view's width must be a multiple of {TILE_WIDTH}, got {camera_info.camera_width}")

    def _check_ortho(self, camera_info, lens_coefficients=None, rolling_shutter_motion=None, exposure_motion=None,
                     defocus_parameters=None) -> None:
        """``ValueError`` for what an orthographic view does not combine with (include/gsb200.h): the lens-coefficient,
        rolling-shutter, motion-blur and defocus gradients and records, and the view-parallel exchange.  The 3D filter with
        camera-parameter gradients is refused by ``_check_filter_3d``."""
        for name, on in (("differentiable_distortion", self.differentiable_distortion),
                         ("differentiable_rolling_shutter", self.differentiable_rolling_shutter),
                         ("differentiable_motion_blur", self.differentiable_motion_blur),
                         ("differentiable_defocus", self.differentiable_defocus),
                         ("a gradient_exchange", self.gradient_exchange is not None),
                         ("a rolling shutter (camera_info.rolling_shutter)", getattr(camera_info, "rolling_shutter", None) is not None),
                         ("motion blur (camera_info.motion_blur)", getattr(camera_info, "motion_blur", None) is not None),
                         ("defocus (camera_info.defocus)", getattr(camera_info, "defocus", None) is not None),
                         ("lens_coefficients", lens_coefficients is not None),
                         ("rolling_shutter_motion", rolling_shutter_motion is not None),
                         ("exposure_motion", exposure_motion is not None),
                         ("defocus_parameters", defocus_parameters is not None)):
            if on:
                raise ValueError(f"an orthographic camera is not supported with {name}")

    def _rolling_shutter_args(self, camera_info, motion=None) -> Optional[_lib.GsbRollingShutterArgs]:
        """The C rolling-shutter argument of ``camera_info.rolling_shutter`` (None: the global-shutter kernels; row_time is
        set by the caller), after the checks of the options a rolling shutter does not combine with; with ``motion``
        (``differentiable_rolling_shutter``) its values replace the record's (read on the host: free for a CPU tensor, one
        blocking 24-byte copy for a device tensor)."""
        rolling_shutter = getattr(camera_info, "rolling_shutter", None)
        if motion is not None:
            if not self.differentiable_rolling_shutter:
                raise ValueError("rolling_shutter_motion needs differentiable_rolling_shutter=True")
            if rolling_shutter is None:
                raise ValueError("rolling_shutter_motion was given for a camera without a rolling shutter "
                                 "(camera_info.rolling_shutter is None)")
        if rolling_shutter is None:
            return None
        for name, on in (("differentiable_pose", self.differentiable_pose),
                         ("differentiable_intrinsics", self.differentiable_intrinsics),
                         ("differentiable_distortion", self.differentiable_distortion),
                         ("a gradient_exchange", self.gradient_exchange is not None)):
            if on:
                raise ValueError(f"a rolling-shutter camera is not supported with {name}")
        values = rolling_shutter.motion
        if motion is not None:
            if not isinstance(motion, torch.Tensor):
                raise ValueError("rolling_shutter_motion must be a torch.Tensor")
            if tuple(motion.shape) != (6,):
                raise ValueError(f"rolling_shutter_motion must have shape (6,), got {tuple(motion.shape)}")
            if motion.dtype != torch.float32:
                raise ValueError(f"rolling_shutter_motion must be float32, got {motion.dtype}")
            values = motion.detach().cpu().tolist()
            if not all(math.isfinite(v) for v in values):
                raise ValueError(f"rolling_shutter_motion must be finite, got {values}")
        return _lib.GsbRollingShutterArgs(motion=(ctypes.c_float * 6)(*values), row_time=None)

    def _motion_blur_args(self, camera_info, motion=None, rolling_shutter_motion=None,
                          point_filter_3d=None) -> Optional[_lib.GsbMotionBlurArgs]:
        """The C motion-blur argument of ``camera_info.motion_blur`` (None: the kernels without blur), after the checks of
        the options a motion blur does not combine with; with ``motion`` (``differentiable_motion_blur``) its values replace
        the record's (read on the host like ``rolling_shutter_motion``)."""
        motion_blur = getattr(camera_info, "motion_blur", None)
        if motion is not None:
            if not self.differentiable_motion_blur:
                raise ValueError("exposure_motion needs differentiable_motion_blur=True")
            if motion_blur is None:
                raise ValueError("exposure_motion was given for a camera without motion blur (camera_info.motion_blur is None)")
        if motion_blur is None:
            return None
        for name, on in (("differentiable_pose", self.differentiable_pose),
                         ("differentiable_intrinsics", self.differentiable_intrinsics),
                         ("differentiable_distortion", self.differentiable_distortion),
                         ("a gradient_exchange", self.gradient_exchange is not None),
                         ("point_filter_3d", point_filter_3d is not None),
                         ("rolling_shutter_motion (one motion gradient per call)", rolling_shutter_motion is not None)):
            if on:
                raise ValueError(f"a motion-blurred camera is not supported with {name}")
        values = motion_blur.motion
        if motion is not None:
            if not isinstance(motion, torch.Tensor):
                raise ValueError("exposure_motion must be a torch.Tensor")
            if tuple(motion.shape) != (6,):
                raise ValueError(f"exposure_motion must have shape (6,), got {tuple(motion.shape)}")
            if motion.dtype != torch.float32:
                raise ValueError(f"exposure_motion must be float32, got {motion.dtype}")
            values = motion.detach().cpu().tolist()
            if not all(math.isfinite(v) for v in values):
                raise ValueError(f"exposure_motion must be finite, got {values}")
        return _lib.GsbMotionBlurArgs(motion=(ctypes.c_float * 6)(*values))

    def _defocus_args(self, camera_info, parameters=None, rolling_shutter_motion=None, point_filter_3d=None,
                      exposure_motion=None) -> Optional[_lib.GsbDefocusArgs]:
        """The C defocus argument of ``camera_info.defocus`` (None: the kernels without defocus), after the checks of the
        options a defocus does not combine with; with ``parameters`` (``differentiable_defocus``) its values (a, rho) replace
        the record's (read on the host like ``exposure_motion``)."""
        defocus = getattr(camera_info, "defocus", None)
        if parameters is not None:
            if not self.differentiable_defocus:
                raise ValueError("defocus_parameters needs differentiable_defocus=True")
            if defocus is None:
                raise ValueError("defocus_parameters was given for a camera without defocus (camera_info.defocus is None)")
        if defocus is None:
            return None
        for name, on in (("differentiable_pose", self.differentiable_pose),
                         ("differentiable_intrinsics", self.differentiable_intrinsics),
                         ("differentiable_distortion", self.differentiable_distortion),
                         ("a gradient_exchange", self.gradient_exchange is not None),
                         ("point_filter_3d", point_filter_3d is not None),
                         ("rolling_shutter_motion (one camera gradient per call)", rolling_shutter_motion is not None),
                         ("exposure_motion (one camera gradient per call)", exposure_motion is not None)):
            if on:
                raise ValueError(f"a defocused camera is not supported with {name}")
        values = defocus.parameters
        if parameters is not None:
            if not isinstance(parameters, torch.Tensor):
                raise ValueError("defocus_parameters must be a torch.Tensor")
            if tuple(parameters.shape) != (2,):
                raise ValueError(f"defocus_parameters must have shape (2,), got {tuple(parameters.shape)}")
            if parameters.dtype != torch.float32:
                raise ValueError(f"defocus_parameters must be float32, got {parameters.dtype}")
            values = parameters.detach().cpu().tolist()
            if not all(math.isfinite(v) for v in values):
                raise ValueError(f"defocus_parameters must be finite, got {values}")
        return _lib.GsbDefocusArgs(aperture=values[0], inverse_focus=values[1])

    # ------------------------------------------------------------------ backward plumbing
    def _run_backward(self, ctx, grad_rasterized_image, grad_rasterized_depth=None, grad_pixel_accumulated_alpha=None,
                      grad_feature_map=None, pose=False, camera_grads=()):
        """The gradients by input slot: dL/dxyz, dL/dfeatures, for a call with extra features dL/d of them ((N, C); zeros
        when the feature map was not used), with ``pose`` dL/dq_pointcloud_camera (K, 4) and dL/dt_pointcloud_camera
        (K, 3), and for each slot of ``camera_grads`` (``_CAMERA_GRADS``) that tensor's gradient: K's (3, 3), the others
        sliced to the tensor's length on its device."""
        cfg = self.config
        lib = _lib.load()
        (pointcloud, pointcloud_features, point_object_id, q_pointcloud_camera, t_pointcloud_camera, K, acc_alpha,
         last_effective, ws, depth, extra_features) = ctx.saved_tensors
        # differentiable_depth: the depth gradient (None when the loss does not use depth) and the forward's depth map
        if grad_rasterized_depth is None:
            depth = None
        camera: _Camera = ctx.camera
        frame: Frame = ctx.frame
        device = pointcloud.device
        N = pointcloud.shape[0]
        M = frame.num_points_in_camera
        H, W = frame.height, frame.width
        band = ctx.color_max_sh_band
        band_i = int(band) if band in (0, 1, 2) else 3  # GPCR:1167-1182: anything else clears nothing
        with torch.cuda.device(device):
            stream = torch.cuda.current_stream(device)
            grad_image = grad_rasterized_image.contiguous()
            if grad_image.dtype != torch.float32:
                grad_image = grad_image.float()
            # both dense gradients live in ONE allocation (xyz rows, pad to 16 B, feature rows) so that a
            # view-parallel trainer can sum them over ranks with a single collective (parallel.py)
            off = (3 * N + 3) // 4 * 4
            flat = torch.empty((off + 56 * N,), dtype=torch.float32, device=device)
            if off > 3 * N:
                flat[3 * N:off].zero_()
            grad_pointcloud = flat[:3 * N].view(N, 3)
            grad_pointcloud_features = flat[off:off + 56 * N].view(N, 56)
            self.last_gradient_buffer = flat
            accum = torch.empty((max(M, 1), _ACCUM_FLOATS), dtype=torch.float32, device=device)
            magnitude_on_image = torch.empty((H, W, 2), dtype=torch.float32, device=device)
            t_pc = t_pointcloud_camera.contiguous()
            backward_flags = self.backward_flags(frame.flags)
            exchange = self.gradient_exchange
            compact = exchange is not None and exchange.world > 1
            grad_sum = blocks = None
            if compact:
                n_obj = ctx.num_objects
                grad_sum, blocks = exchange.allocate(N, n_obj, device)
                blocks[exchange.rank, 3 * N:3 * N + 3 * n_obj] = t_pc.reshape(-1)
                backward_flags |= _lib.GSB_FLAG_COMPACT_GRADS
            args = _lib.GsbBackwardArgs(
                num_points=N, pointcloud=_ptr(pointcloud), pointcloud_features=_ptr(pointcloud_features),
                point_object_id=_ptr(point_object_id), num_objects=ctx.num_objects,
                t_pointcloud_camera=_ptr(t_pc), camera_intrinsics=_ptr(K), camera_height=H, camera_width=W,
                far_plane=cfg.far_plane, depth_to_sort_key_scale=cfg.depth_to_sort_key_scale,
                color_max_sh_band=band_i, grad_q_factor=cfg.grad_q_factor, grad_s_factor=cfg.grad_s_factor,
                grad_alpha_factor=cfg.grad_alpha_factor, grad_color_factor=cfg.grad_color_factor,
                grad_high_order_color_factor=cfg.grad_high_order_color_factor, flags=backward_flags,
                workspace=_ptr(ws), workspace_bytes=frame.layout.total_bytes, key_capacity=frame.key_capacity,
                grad_rasterized_image=_ptr(grad_image), pixel_accumulated_alpha=_ptr(acc_alpha),
                pixel_offset_of_last_effective_point=_ptr(last_effective), accum=_ptr(accum),
                accum_rows=M, grad_pointcloud=_ptr(grad_pointcloud),
                grad_pointcloud_features=_ptr(grad_pointcloud_features),
                magnitude_grad_viewspace_on_image=_ptr(magnitude_on_image), stream=stream.cuda_stream,
                grad_sum_compact=_ptr(grad_sum), grad_color_compact=_ptr(blocks[exchange.rank]) if compact else None)
            grad_depth = _f32(grad_rasterized_depth) if depth is not None else None
            # differentiable_alpha: None when the loss does not use the accumulated alpha
            grad_alpha = _f32(grad_pixel_accumulated_alpha) if self.differentiable_alpha else None
            grads = {_XYZ: grad_pointcloud, _FEATURES: grad_pointcloud_features}
            ext = None
            if extra_features is not None:  # dL/df: written by the call, or zero when the feature map was not used
                C = extra_features.shape[1]
                if grad_feature_map is None:
                    grads[_EXTRA_FEATURES] = torch.zeros((N, C), dtype=torch.float32, device=device)
                else:
                    grads[_EXTRA_FEATURES] = torch.empty((N, C), dtype=torch.float32, device=device)
                    grad_map = _f32(grad_feature_map)
                    ext = _lib.GsbExtraFeatureArgs(channels=C, features=_ptr(extra_features), grad_rasterized=_ptr(grad_map),
                                                   grad_features=_ptr(grads[_EXTRA_FEATURES]))
            temps = []  # the camera-gradient temps, alive until the call returns
            pose_args = None
            if pose:
                n_obj = ctx.num_objects
                q_pc = q_pointcloud_camera.detach().contiguous()
                grads[_Q] = torch.empty((n_obj, 4), dtype=torch.float32, device=device)
                grads[_T] = torch.empty((n_obj, 3), dtype=torch.float32, device=device)
                temps.append(torch.empty((max(int(lib.gsb200_pose_grad_temp_bytes(n_obj)), 16) // 4,), dtype=torch.float32,
                                         device=device))
                pose_args = _lib.GsbPoseGradArgs(q_pointcloud_camera=_ptr(q_pc), grad_q_pointcloud_camera=_ptr(grads[_Q]),
                                                 grad_t_pointcloud_camera=_ptr(grads[_T]), temp=_ptr(temps[-1]))
            grad_args = dict.fromkeys(_CAMERA_GRADS)
            for slot in camera_grads:
                struct, shape, temp_bytes = _CAMERA_GRADS[slot]
                grads[slot] = torch.empty(shape, dtype=torch.float32, device=device)
                temps.append(torch.empty((int(getattr(lib, temp_bytes)()) // 4,), dtype=torch.float32, device=device))
                grad_args[slot] = struct(_ptr(grads[slot]), _ptr(temps[-1]))
            # backward_impl's precedence (csrc/api.cu): every refused combination was refused by _resolve_camera
            if camera.projection is _EQUIRECT:
                entry, camera_args = "gsb200_backward_equirect", ()
            elif camera.projection is _ORTHO:
                entry, camera_args = "gsb200_backward_ortho", (camera.filter_3d, pose_args, grad_args[_INTRINSICS])
            elif camera.defocus is not None:
                entry, camera_args = "gsb200_backward_defocus", (camera.lens, camera.rolling_shutter, camera.motion_blur,
                                                                 camera.defocus, grad_args[_DEFOCUS_PARAMETERS])
            elif camera.motion_blur is not None:
                entry, camera_args = "gsb200_backward_motion_blur", (camera.lens, camera.rolling_shutter, camera.motion_blur,
                                                                     grad_args[_EXPOSURE_MOTION])
            elif camera.filter_3d is not None:
                entry, camera_args = "gsb200_backward_filter3d", (camera.lens, camera.rolling_shutter, camera.filter_3d)
            elif camera.rolling_shutter is not None:
                entry, camera_args = "gsb200_backward_rolling_shutter", (camera.lens, camera.rolling_shutter,
                                                                         grad_args[_ROLLING_SHUTTER_MOTION])
            elif camera.lens is not None:
                entry, camera_args = "gsb200_backward_lens_calib", (camera.lens, grad_args[_LENS_COEFFICIENTS], pose_args,
                                                                    grad_args[_INTRINSICS])
            else:
                entry, camera_args = "gsb200_backward_calib", (pose_args, grad_args[_INTRINSICS])
            _lib.check(getattr(lib, entry)(ctypes.byref(args), _ptr(grad_depth), _ptr(depth), _ptr(grad_alpha), _ref(ext),
                                           *map(_ref, camera_args)), entry)
            for slot, (length, like_device) in camera.gradient_like.items():
                if slot in grads:
                    grads[slot] = grads[slot][:length].to(like_device)
            own_view_grad_xyz = None
            if compact:
                exchange.rows_written(grad_sum, blocks)
                if self.backward_valid_point_hook is not None:  # the hook sees this rank's own view (before the sum)
                    own_view_grad_xyz = grad_sum[frame.point_id_in_camera_list.long(), 0:3]

                def expand(part: int) -> None:
                    """Dense gradients from the exchanged compact rows, on the CURRENT stream (part 0: everything; 1: the SH
                    columns, which need only the gathered blocks; 2: the summed columns) -- csrc/blend_bwd.cu."""
                    eargs = _lib.GsbExpandArgs(
                        num_points=N, num_views=exchange.world, num_objects=ctx.num_objects, grad_sum=_ptr(grad_sum),
                        grad_color_views=_ptr(blocks), view_stride=blocks.shape[1], pointcloud=_ptr(pointcloud),
                        point_object_id=_ptr(point_object_id), color_max_sh_band=band_i,
                        grad_color_factor=cfg.grad_color_factor,
                        grad_high_order_color_factor=cfg.grad_high_order_color_factor, part=part,
                        grad_pointcloud=_ptr(grad_pointcloud), grad_pointcloud_features=_ptr(grad_pointcloud_features),
                        stream=torch.cuda.current_stream(device).cuda_stream)
                    _lib.check(lib.gsb200_expand_view_gradients(ctypes.byref(eargs)), "gsb200_expand_view_gradients")

                exchange.run_and_expand(grad_sum, blocks, expand)

            hook = self.backward_valid_point_hook
            if hook is not None:  # GPCR:1127-1142
                ids = frame.point_id_in_camera_list
                ids64 = ids.long()
                acc = accum[:M]
                hook(GaussianPointCloudRasterisation.BackwardValidPointHookInput(
                    point_id_in_camera_list=ids,
                    grad_point_in_camera=own_view_grad_xyz if compact else grad_pointcloud[ids64],
                    grad_pointfeatures_in_camera=None if compact else grad_pointcloud_features[ids64],
                    grad_viewspace=acc[:, 0:2].contiguous(),
                    magnitude_grad_viewspace=acc[:, 9].contiguous(),
                    magnitude_grad_viewspace_on_image=magnitude_on_image,
                    num_overlap_tiles=frame.num_overlap_tiles,
                    num_affected_pixels=acc[:, 10].round().to(torch.int32),
                    point_uv_in_camera=frame.point_uv.contiguous(),
                    point_depth=frame.records[:, 7] if camera.projection is _EQUIRECT else frame.point_in_camera[:, 2],
                ))
        return grads

    def backward_flags(self, frame_flags: int) -> int:
        """Flags of the backward call for a frame rendered with ``frame_flags`` (adds the experimental kernel selection)."""
        if self.backward_impl == "transposed":
            frame_flags |= _lib.GSB_FLAG_BACKWARD_TRANSPOSED
        if self.backward_valid_point_hook is None and (self.backward_impl == "transposed" or self.skip_unused_hook_statistics):
            frame_flags |= _lib.GSB_FLAG_NO_HOOK_STATS  # the reference's need_extra_info = False, GPCR:521
        return frame_flags

    # ------------------------------------------------------------------ public forward (GPCR:1184-1204)
    def forward(self, input_data: "GaussianPointCloudRasterisation.GaussianPointCloudRasterisationInput",
                point_extra_features: Optional[torch.Tensor] = None, lens_coefficients: Optional[torch.Tensor] = None,
                rolling_shutter_motion: Optional[torch.Tensor] = None, point_filter_3d: Optional[torch.Tensor] = None,
                exposure_motion: Optional[torch.Tensor] = None, defocus_parameters: Optional[torch.Tensor] = None):
        """Returns (image, depth, pixel_valid_point_count), then pixel_accumulated_alpha with ``differentiable_alpha``.
        ``point_extra_features`` (an extension): an (N, C) float32 tensor of per-Gaussian values (1 <= C <= 16; semantic
        logits, instance encodings, distilled features, ...), contiguous, on the scene's device.  The output tuple then
        ends with their blend ``F_p = sum_i alpha_i T_i f_i``, (H, W, C) float32, with exactly the image's weights: no
        normalisation, no background, no activation.  It is differentiable in the features (dL/dF rows of points outside
        the frustum are zero, no gradient factor) and, through the weights, in xyz, q, s and the opacity, as the image is;
        the backward runs for the features alone too.  Combines with ``differentiable_depth`` and ``differentiable_alpha``.
        ``ValueError`` with ``backward_impl="butterfly"``, ``config.rgb_only``, a ``gradient_exchange``, or a tensor of the
        wrong shape, dtype, device or layout.  The densification controller does not know these rows: a caller who clones,
        splits or removes Gaussians must keep ``point_extra_features`` in step.
        ``input_data.camera_info.distortion`` (an extension; ``Camera.LensDistortion``): render and differentiate through
        an OpenCV radial-tangential or fisheye lens (``gsb200_forward_lens`` / ``gsb200_backward_lens``; definition in
        ``include/gsb200.h``).  Every output and option above works with a lens, except ``differentiable_pose``,
        ``differentiable_intrinsics`` (both allowed with ``camera_gradients_through_lens``, ``gsb200_backward_lens_calib``)
        and a ``gradient_exchange`` (``ValueError``).
        ``lens_coefficients`` (with ``differentiable_distortion``; an extension): a float32 tensor of the lens model's length
        (5 for ``opencv``, 4 for ``fisheye``), on any device.  Its values are the coefficients rendered (``camera_info.
        distortion`` supplies the model), and the backward returns dL/d ``lens_coefficients`` on the tensor's device.  The
        values are read on the host: free for a CPU tensor, one blocking 20-byte copy for a device tensor.  ``ValueError``
        for a camera with no lens, a tensor of the wrong length or dtype, or an operator without the option.  None: no
        coefficient gradient.
        ``input_data.camera_info.rolling_shutter`` (an extension; ``Camera.RollingShutter``): render and differentiate each
        point at its row time through the view's motion (``gsb200_forward_rolling_shutter`` /
        ``gsb200_backward_rolling_shutter``; definition in ``include/gsb200.h``), with or without a lens.  ``last_frame``'s
        ``point_in_camera`` and ``point_uv`` are the values at each point's row time.  Every output and option above works
        with a rolling shutter, except ``differentiable_pose``, ``differentiable_intrinsics``, ``differentiable_distortion``
        and a ``gradient_exchange`` (``ValueError``).
        ``rolling_shutter_motion`` (with ``differentiable_rolling_shutter``; an extension): a (6,) float32 tensor (v, w) on
        any device.  Its values are the motion rendered, and the backward returns dL/d ``rolling_shutter_motion`` on the
        tensor's device.  The values are read on the host like ``lens_coefficients``.  ``ValueError`` for a camera without
        a rolling shutter, a tensor of the wrong shape or dtype, or an operator without the option.  None: no motion
        gradient.
        ``point_filter_3d`` (an extension; ``mip_filter.compute_filter_3d``): an (N,) float32 tensor of per-Gaussian 3D
        smoothing filter stds sigma >= 0, contiguous, on the scene's device.  Every Gaussian is rendered convolved with an
        isotropic Gaussian of std sigma: scales sqrt(exp(s)^2 + sigma^2) and opacity o times the compensation c
        (``gsb200_forward_filter3d`` / ``gsb200_backward_filter3d``; definition in ``include/gsb200.h``); the stored rows are
        not changed, and the gradients are with respect to them.  The filter gets no gradient.  Works with extra features,
        depth, alpha, every lens, a rolling shutter and either backward kernel for an image-only loss.  ``ValueError`` with
        ``differentiable_pose``, ``differentiable_intrinsics``, ``differentiable_distortion``,
        ``differentiable_rolling_shutter``, a ``gradient_exchange``, ``lens_coefficients``, ``rolling_shutter_motion``, or a
        tensor of the wrong shape, dtype, device or layout.
        ``input_data.camera_info.motion_blur`` (an extension; ``Camera.MotionBlur``): render and differentiate the view with
        each splat widened by its screen motion over the exposure (``gsb200_forward_motion_blur`` /
        ``gsb200_backward_motion_blur``; definition in ``include/gsb200.h``), with or without a lens and a rolling shutter.
        Every output and option above works with it, except ``differentiable_pose``, ``differentiable_intrinsics``,
        ``differentiable_distortion``, a ``gradient_exchange``, ``point_filter_3d`` and ``rolling_shutter_motion``
        (``ValueError``).  A sharp render of the same view is the camera with ``motion_blur=None``.
        ``exposure_motion`` (with ``differentiable_motion_blur``; an extension): a (6,) float32 tensor (v, w) on any device.
        Its values are the exposure motion rendered, and the backward returns dL/d ``exposure_motion`` on the tensor's
        device.  ``ValueError`` for a camera without motion blur, a tensor of the wrong shape or dtype, or an operator without
        the option.  None: no motion gradient.
        ``input_data.camera_info.defocus`` (an extension; ``Camera.Defocus``): render and differentiate the view through a
        thin lens, each splat widened by its defocus blur (``gsb200_forward_defocus`` / ``gsb200_backward_defocus``;
        definition in ``include/gsb200.h``), with or without a lens, a rolling shutter and motion blur.  Every output and
        option above works with it, except ``differentiable_pose``, ``differentiable_intrinsics``,
        ``differentiable_distortion``, a ``gradient_exchange``, ``point_filter_3d``, ``rolling_shutter_motion`` and
        ``exposure_motion`` (``ValueError``).  A pinhole render of the same view is the camera with ``defocus=None``; a
        refocused one is the camera with another ``Defocus``.
        ``defocus_parameters`` (with ``differentiable_defocus``; an extension): a (2,) float32 tensor (a, rho) on any
        device.  Its values are the aperture and inverse focus distance rendered (a negative a renders as |a|), and the
        backward returns dL/d ``defocus_parameters`` on the tensor's device.  ``ValueError`` for a camera without defocus, a
        tensor of the wrong shape or dtype, or an operator without the option.  None: no defocus gradient.
        ``camera_info.distortion = LensDistortion("orthographic", ())`` (an extension): render and differentiate a parallel
        projection (``gsb200_forward_ortho`` / ``gsb200_backward_ortho``; definition in ``include/gsb200.h``).  Depth is z,
        and the SH colour is seen along the camera's forward axis.  Works with extra features, depth, alpha,
        ``differentiable_pose``, ``differentiable_intrinsics``, ``point_filter_3d`` (not with the two camera gradients) and
        either backward kernel for an image-only loss.  ``ValueError``, before any device work, with
        ``differentiable_distortion``, ``differentiable_rolling_shutter``, ``differentiable_motion_blur``,
        ``differentiable_defocus``, a ``gradient_exchange``, a rolling shutter, motion blur or defocus on the camera, or their
        tensors."""
        camera_info = input_data.camera_info
        return self._module_function.apply(
            input_data.point_cloud, input_data.point_cloud_features, input_data.point_invalid_mask,
            input_data.point_object_id, input_data.q_pointcloud_camera, input_data.t_pointcloud_camera, camera_info,
            input_data.color_max_sh_band, point_extra_features,
            camera_info.camera_intrinsics if self.differentiable_intrinsics else None, lens_coefficients,
            rolling_shutter_motion, point_filter_3d, exposure_motion, defocus_parameters)


@dataclass
class GaussianPoint3D:
    """The fields of the reference's ``GaussianPoint3D`` Taichi struct (GaussianPoint3D.py:17-27) as tensors."""
    translation: torch.Tensor  # (3,)
    cov_rotation: torch.Tensor  # (4,) xyzw
    cov_scale: torch.Tensor  # (3,) log-scale
    alpha: torch.Tensor  # () opacity logit
    color_r: torch.Tensor  # (16,)
    color_g: torch.Tensor  # (16,)
    color_b: torch.Tensor  # (16,)


def load_point_cloud_row_into_gaussian_point_3d(pointcloud: torch.Tensor, pointcloud_features: torch.Tensor,
                                                point_id: int) -> GaussianPoint3D:
    """Same name, arguments and row layout as the reference's ``@ti.func`` (GPCR:208-236; imported by its controller,
    GaussianPointAdaptiveController.py:4, and pinned by its test ``test_load_point_cloud_row_into_gaussian_point_3d``):
    row ``point_id`` of the (N,3) / (N,56) tensors as a ``GaussianPoint3D`` -- q xyzw | log-scale | opacity logit |
    R, G, B SH x 16.  Host-side views; inside the kernels the same split is done by ``preprocess_kernel``."""
    f = pointcloud_features[point_id]
    return GaussianPoint3D(translation=pointcloud[point_id], cov_rotation=f[0:4], cov_scale=f[4:7], alpha=f[7],
                           color_r=f[8:24], color_g=f[24:40], color_b=f[40:56])


def find_tile_start_and_end(point_in_camera_sort_key: torch.Tensor, tile_points_start: torch.Tensor,
                            tile_points_end: torch.Tensor) -> None:
    """Same call shape as the reference kernel (GPCR:175-193; used by its tests): sorted int64 keys
    ``tile << 32 | depth`` -> per-tile [start, end) written into the two zero-initialised int32 outputs."""
    lib = _lib.load()
    _require(point_in_camera_sort_key, "point_in_camera_sort_key", torch.int64)
    _require(tile_points_start, "tile_points_start", torch.int32)
    _require(tile_points_end, "tile_points_end", torch.int32)
    fn = lib.gsb200_find_tile_start_and_end
    with torch.cuda.device(point_in_camera_sort_key.device):
        stream = torch.cuda.current_stream(point_in_camera_sort_key.device)
        keys = point_in_camera_sort_key.contiguous()
        _lib.check(fn(keys.data_ptr(), keys.shape[0], tile_points_start.data_ptr(), tile_points_end.data_ptr(),
                      tile_points_start.shape[0], stream.cuda_stream), "gsb200_find_tile_start_and_end")
