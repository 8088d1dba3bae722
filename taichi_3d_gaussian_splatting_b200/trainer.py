"""Training step around the operator (SURVEY §8(f)-2; BASELINE config 5 harness).

A compact mirror of the reference loop ``GaussianPointCloudTrainer.train``
(``taichi_3d_gaussian_splatting/GaussianPointTrainer.py:118-267``) for in-memory datasets: two Adam
optimisers (features / positions, :126-129), exponential decay of the position LR every
``position_learning_rate_decay_interval`` iterations (:131-132, 182-183), image down-sampling schedule
4 -> 2 -> 1 with the crop-to-16 rule (:98-116, 139-148), SH band schedule ``it // interval`` (:164),
clamp + HWC->CHW + ``LossFunction`` (:168-175), controller ``refinement`` after the optimiser step (:194).
TensorBoard logging, the parquet/JSON dataset and validation image dumps are out of scope.
Optional supervision (an extension; ``TrainConfig.depth_loss_weight`` / ``mask_loss_weight`` / ``background``, per-view
``SupervisionTargets`` as a fifth view element): a masked-L1 depth loss, an L1 mask loss on the accumulated alpha and
training on a white or random background, with the same loss (``loss.supervision_loss``) in the autograd loop and in the
fused step.
Optional feature training (an extension; ``Scene.point_extra_features``, ``TrainConfig.feature_loss``, per-view
``SupervisionTargets.labels`` / ``features``): per-Gaussian feature vectors rendered alongside the image, a cross-entropy or
l2 loss on the rendered feature map (``loss.feature_loss``) and a third Adam on the features, kept in step with the scene
through densification.
Optional pose refinement (an extension; ``TrainConfig.pose_learning_rate``): the (q, t) of every training view but the
first become trainable, differentiated by the operator's ``differentiable_pose`` and stepped by their own Adam.
Optional intrinsics refinement (an extension; ``TrainConfig.intrinsics_learning_rate``): per camera, a correction of the focal
lengths and the principal point, differentiated by the operator's ``differentiable_intrinsics`` and stepped by its own Adam.
Views with lens distortion (an extension; ``CameraInfo.distortion``) train through their lens in the autograd loop; the
downsampled camera keeps the coefficients (they act on the normalised image plane).  Not with ``fused_step``, pose or
intrinsics refinement.
Optional lens refinement (an extension; ``TrainConfig.distortion_learning_rate``): per camera with a lens, its coefficients,
differentiated by the operator's ``differentiable_distortion`` and stepped by their own Adam.
Views with a rolling shutter (an extension; ``CameraInfo.rolling_shutter``) train through it in the autograd loop; the
downsampled camera keeps the motion (row time is normalised by the image height).  Not with ``fused_step``, pose, intrinsics
or lens refinement.  Optional motion refinement (``TrainConfig.rolling_shutter_learning_rate``): per rolling-shutter view, its
motion (v, w), differentiated by the operator's ``differentiable_rolling_shutter`` and stepped by its own Adam.
Optional appearance compensation (an extension; ``TrainConfig.appearance_grid``): one bilateral grid per training view
(``appearance.apply_bilateral_grid``), initialised to the identity, slices the image the image loss sees (after the
background composite), with a TV prior and its own Adam that steps only the visited view's grid.  It acts on the image alone,
so it composes with every other option; ``validation`` renders the raw image (a held-out view has no grid).
Optional MCMC densification (an extension; ``TrainConfig.densification="mcmc"``, ``mcmc_config``): the scene grows to a
fixed budget by relocating dead Gaussians and adding 5 % per refinement (``mcmc.GaussianPointMCMCController``), with the
opacity and scale regularisers in the loss and a covariance-shaped position noise after the optimiser step.  The adaptive
controller and the backward hook are then not used.  Not with the optional scale regulariser of the loss function nor with a
view-parallel gradient exchange.
Optional per-pixel weights of the image loss (an extension; ``TrainConfig.robust_loss``, per-view
``SupervisionTargets.loss_weight``): transient distractors (people, cars, shadows in one view only) are dropped from the
image loss by RobustNeRF's trimmed inlier mask of each iteration's residual and / or by a static weight per view
(``loss.robust_weight``), in the autograd loop (torch form, inside the appearance grid's wrapper) and in the fused step
(``gsb200_train_step_robust``).  The depth, mask and feature terms are not weighted; ``validation`` is unchanged.  Not with
the view-parallel gradient exchange.
The rasteriser is injected (default: the CUDA operator) so that tests can run the identical loop with the
CPU oracle behind the same interface and compare PSNR trajectories.
"""
import math
from dataclasses import dataclass, field
from typing import Callable, List, Optional, Tuple

import torch
import torch.nn.functional as F

from .appearance import apply_bilateral_grid, bilateral_grid_tv, check_grid_shape, identity_grids
from .Camera import CameraInfo, LensDistortion, RollingShutter
from .densification import GaussianPointAdaptiveController
from .GaussianPointCloudRasterisation import GaussianPointCloudRasterisation
from .loss import (FEATURE_LOSSES, LossFunction, RobustLossConfig, SupervisionTargets, feature_loss, mcmc_regulariser,
                   robust_composite, robust_weight, supervision_loss)
from .mcmc import GATE_K, GaussianPointMCMCController, MCMCConfig, MCMCMoments, add_position_noise
from .mip_filter import compute_filter_3d

View = Tuple[torch.Tensor, torch.Tensor, torch.Tensor, CameraInfo]  # image (3,H,W) in [0,1], q (1,4), t (1,3), camera
# ... optionally followed by a SupervisionTargets (depth and / or mask at the image's resolution)
BACKGROUNDS = ("black", "white", "random")
DENSIFICATIONS = ("adaptive", "mcmc")


def psnr(pred: torch.Tensor, target: torch.Tensor) -> float:
    mse = torch.mean((pred.clamp(0, 1) - target) ** 2).item()
    return float("inf") if mse == 0 else -10.0 * math.log10(mse)


def downsample_image_and_camera_info(image: torch.Tensor, camera_info: CameraInfo, downsample_factor: int):
    """GaussianPointTrainer.py:98-116: antialiased resize, crop to multiples of 16, scale fx fy cx cy."""
    h = camera_info.camera_height // downsample_factor
    w = camera_info.camera_width // downsample_factor
    image = F.interpolate(image[None], size=(h, w), mode="bilinear", antialias=True, align_corners=False)[0]
    w -= w % 16
    h -= h % 16
    image = image[:3, :h, :w].contiguous()
    K = camera_info.camera_intrinsics.clone()
    K[0, 0] /= downsample_factor
    K[1, 1] /= downsample_factor
    K[0, 2] /= downsample_factor
    K[1, 2] /= downsample_factor
    # the lens coefficients act on the normalised image plane and row time is normalised by the height: resizing changes
    # neither the lens nor the rolling-shutter motion
    return image, CameraInfo(camera_intrinsics=K, camera_height=h, camera_width=w, camera_id=camera_info.camera_id,
                             distortion=camera_info.distortion, rolling_shutter=camera_info.rolling_shutter)


def _nearest(x: torch.Tensor, h: int, w: int, hc: int, wc: int) -> torch.Tensor:
    """(H, W, ...) -> (hc, wc, ...): the rows and columns ``F.interpolate(mode="nearest")`` picks for an (h, w) output,
    cropped; exact for any dtype (the indices are resized, not the values)."""
    rows = F.interpolate(torch.arange(x.shape[0], dtype=torch.float32, device=x.device)[None, None], size=h,
                         mode="nearest")[0, 0, :hc].long()
    cols = F.interpolate(torch.arange(x.shape[1], dtype=torch.float32, device=x.device)[None, None], size=w,
                         mode="nearest")[0, 0, :wc].long()
    return x[rows][:, cols].contiguous()


def downsample_targets(targets: SupervisionTargets, camera_info: CameraInfo, downsample_factor: int) -> SupervisionTargets:
    """The targets of a view at the schedule's resolution: the mask and the loss weight with the image's antialiased resize,
    the depth, the labels and the feature map with nearest neighbour (a sparse map stays sparse, nothing is blended across
    an edge); all cropped like the image."""
    h = camera_info.camera_height // downsample_factor
    w = camera_info.camera_width // downsample_factor
    hc, wc = h - h % 16, w - w % 16
    mask = depth = None
    if targets.mask is not None:
        mask = F.interpolate(targets.mask[None, None], size=(h, w), mode="bilinear", antialias=True,
                             align_corners=False)[0, 0, :hc, :wc].contiguous()
    if targets.depth is not None:
        depth = F.interpolate(targets.depth[None, None], size=(h, w), mode="nearest")[0, 0, :hc, :wc].contiguous()
    labels = None if targets.labels is None else _nearest(targets.labels, h, w, hc, wc)
    features = None if targets.features is None else _nearest(targets.features, h, w, hc, wc)
    loss_weight = None
    if targets.loss_weight is not None:
        loss_weight = F.interpolate(targets.loss_weight[None, None], size=(h, w), mode="bilinear", antialias=True,
                                    align_corners=False)[0, 0, :hc, :wc].contiguous()
    return SupervisionTargets(depth=depth, mask=mask, labels=labels, features=features, loss_weight=loss_weight)


@dataclass
class Scene:
    """The trainable tensors of ``GaussianPointCloudScene`` (GaussianPointCloudScene.py:25-60), no IO."""
    point_cloud: torch.Tensor  # (N,3) leaf, requires_grad
    point_cloud_features: torch.Tensor  # (N,56) leaf, requires_grad
    point_invalid_mask: torch.Tensor  # (N,) int8
    point_object_id: torch.Tensor  # (N,) int32
    point_extra_features: Optional[torch.Tensor] = None  # (N, C) leaf, requires_grad: per-Gaussian feature vectors


class GaussianPointCloudTrainer:
    @dataclass
    class TrainConfig:
        # defaults of GaussianPointTrainer.py:32-58
        num_iterations: int = 300000
        feature_learning_rate: float = 1e-3
        position_learning_rate: float = 1e-5
        position_learning_rate_decay_rate: float = 0.97
        position_learning_rate_decay_interval: int = 100
        increase_color_max_sh_band_interval: float = 1000.
        initial_downsample_factor: int = 4
        half_downsample_factor_interval: int = 250
        rasterisation_config: GaussianPointCloudRasterisation.GaussianPointCloudRasterisationConfig = field(
            default_factory=GaussianPointCloudRasterisation.GaussianPointCloudRasterisationConfig)
        adaptive_controller_config: GaussianPointAdaptiveController.GaussianPointAdaptiveControllerConfig = field(
            default_factory=GaussianPointAdaptiveController.GaussianPointAdaptiveControllerConfig)
        loss_function_config: LossFunction.LossFunctionConfig = field(
            default_factory=LossFunction.LossFunctionConfig)
        # optional supervision (loss.supervision_loss): weights of the masked-L1 depth term and of the L1 mask term on the
        # accumulated alpha, and the background the image is composited on ("black" = none, "white", or "random": one
        # colour per iteration, which needs a mask on every view)
        depth_loss_weight: float = 0.
        mask_loss_weight: float = 0.
        background: str = "black"
        # optional feature training (loss.feature_loss): "none", "cross_entropy" (labels) or "l2" (feature maps) on the
        # rendered map of Scene.point_extra_features, its weight (> 0 when on), and the learning rate of the features' own
        # Adam.  The default learning rate is a starting point, not tuned.
        feature_loss: str = "none"
        feature_loss_weight: float = 0.
        extra_feature_learning_rate: float = 1e-2
        # optional pose refinement: > 0 makes the (q, t) of training views 1..n leaf tensors (initialised from the views)
        # trained by their own Adam at this rate, q renormalised after each step.  View 0's pose stays fixed and is the
        # reference frame; the global scale of scene and translations is not pinned.  Not with fused_step.
        pose_learning_rate: float = 0.
        # optional intrinsics refinement: > 0 gives every camera_id of the training views four leaf scalars, initialised to
        # 0 and trained by their own Adam at this rate -- the log-scales of fx and fy, and the offsets of cx and cy in units
        # of the view's full-resolution width and height.  Skew and K[1,0] are not trained.  Combines with
        # pose_learning_rate.  Not with fused_step.
        intrinsics_learning_rate: float = 0.
        # optional lens refinement: > 0 gives every camera_id whose training views have a lens (CameraInfo.distortion) one
        # leaf tensor of its coefficients (5 for opencv, 4 for fisheye), initialised from the views' lens, kept on the host
        # and trained by its own Adam at this rate.  The views of one camera_id must share their lens.  Not with fused_step,
        # pose or intrinsics refinement (no distorted view combines with them).
        distortion_learning_rate: float = 0.
        # optional motion refinement: > 0 gives every training view with a rolling shutter (CameraInfo.rolling_shutter) one
        # (6,) leaf tensor of its motion (v, w), initialised from the view's, kept on the host and trained by its own Adam at
        # this rate.  Not with fused_step, pose, intrinsics or lens refinement (no rolling-shutter view combines with them).
        rolling_shutter_learning_rate: float = 0.
        # optional appearance compensation: (Gx, Gy, Gz) gives every training view one bilateral grid of that many nodes
        # (1 <= Gx, Gy <= 64, 1 <= Gz <= 16; (1, 1, 1) is a per-view affine colour transform), initialised to the identity
        # and trained by its own Adam at appearance_learning_rate with a TV prior of weight appearance_tv_weight.  The
        # defaults are starting points, not tuned.
        appearance_grid: Optional[Tuple[int, int, int]] = None
        appearance_learning_rate: float = 2e-3
        appearance_tv_weight: float = 10.0
        # how the scene grows: "adaptive" (the reference's gradient-threshold controller, adaptive_controller_config) or
        # "mcmc" (relocation, growth to mcmc_config.cap_max, regularisers and position noise; needs mcmc_config)
        densification: str = "adaptive"
        mcmc_config: Optional[MCMCConfig] = None
        # optional 3D smoothing filter (Mip-Splatting, mip_filter.py): every Gaussian is rendered convolved with an isotropic
        # Gaussian sized by the finest sampling interval of the full-resolution training views that see it (variance in
        # pixels^2, the paper's 0.2), recomputed before the first iteration, after every refinement and every
        # mip_filter_interval iterations.  Not with pose, intrinsics, lens or motion refinement, fisheye training views or
        # the view-parallel exchange.  OpenCV-lens and rolling-shutter views use the pinhole test at the mid-readout pose
        # (an approximation).
        mip_filter_3d: bool = False
        mip_filter_variance: float = 0.2
        mip_filter_interval: int = 100
        # optional robust image loss against transient distractors (RobustNeRF's trimmed inlier mask, loss.robust_weight),
        # from robust_loss.start_iteration on.  A view whose targets carry loss_weight is weighted by it in any case.  Not
        # with the view-parallel exchange.
        robust_loss: Optional[RobustLossConfig] = None

    def __init__(self, config: "GaussianPointCloudTrainer.TrainConfig", scene: Scene, train_views: List[View],
                 rasterisation_factory: Optional[Callable] = None, generator: Optional[torch.Generator] = None,
                 fused_image_loss: bool = False, fused_adam: bool = False, fused_controller_update: bool = False,
                 fused_step: bool = False, shuffle_generator: Optional[torch.Generator] = None,
                 background_generator: Optional[torch.Generator] = None):
        """``fused_image_loss``: clamp + L1 + D-SSIM and their gradient in two CUDA kernels (``gsb200_image_loss``)
        instead of ~60 autograd kernels per step; same loss values (CUDA only).  ``fused_adam``: the two Adam updates as
        one kernel each (``optim.FusedAdam`` / ``gsb200_adam_step``) instead of torch's foreach path (CUDA only).
        ``fused_controller_update``: the controller's per-iteration accumulator update as one kernel
        (``gsb200_controller_update``) instead of ~15 torch launches (CUDA only).
        ``fused_step``: the WHOLE iteration as one library call (``gsb200_train_step``: forward, image loss, backward with the
        controller accumulators fused into its epilogue, both Adam updates; no autograd, no host wait; CUDA only).
        ``shuffle_generator``: a CPU ``torch.Generator``; the views are then visited in a fresh random permutation per
        epoch like the reference's shuffling DataLoader (GaussianPointTrainer.py:120-124) instead of in fixed order.
        ``background_generator``: a generator on the scene's device; with ``background="random"`` it draws the colour of
        each iteration on the device (no host wait; the autograd loop and the fused step draw the same colours)."""
        if config.background not in BACKGROUNDS:
            raise ValueError(f"background must be one of {BACKGROUNDS}, got {config.background!r}")
        if config.densification not in DENSIFICATIONS:
            raise ValueError(f"densification must be one of {DENSIFICATIONS}, got {config.densification!r}")
        self._mcmc = config.densification == "mcmc"
        if self._mcmc:
            if not isinstance(config.mcmc_config, MCMCConfig):
                raise ValueError('densification="mcmc" needs mcmc_config (an MCMCConfig with the budget cap_max)')
            config.mcmc_config.check()
            if config.loss_function_config.enable_regularization:
                raise ValueError('densification="mcmc" has its own scale regulariser: switch off '
                                 "loss_function_config.enable_regularization")
        for name in ("depth_loss_weight", "mask_loss_weight"):
            w = getattr(config, name)
            if not (w >= 0.0 and w < float("inf")):
                raise ValueError(f"{name} must be finite and >= 0, got {w}")
        targets = [v[4] if len(v) > 4 and v[4] is not None else SupervisionTargets() for v in train_views]
        if config.depth_loss_weight > 0 and any(tg.depth is None for tg in targets):
            raise ValueError("depth_loss_weight > 0 needs a depth target on every view")
        if config.mask_loss_weight > 0 and any(tg.mask is None for tg in targets):
            raise ValueError("mask_loss_weight > 0 needs a mask on every view")
        if config.background == "random" and any(tg.mask is None for tg in targets):
            raise ValueError('background="random" needs a mask on every view (the ground truth is composited by it)')
        if not (config.pose_learning_rate >= 0.0 and config.pose_learning_rate < float("inf")):
            raise ValueError(f"pose_learning_rate must be finite and >= 0, got {config.pose_learning_rate}")
        self._pose = config.pose_learning_rate > 0
        if self._pose and fused_step:
            raise ValueError("fused_step does not implement pose refinement (pose_learning_rate > 0)")
        # the trainable poses: view 0 keeps its own tensors (the gauge), every other view gets leaf copies
        self._poses = [(v[1], v[2]) if i == 0 or not self._pose else
                       (v[1].detach().clone().requires_grad_(True), v[2].detach().clone().requires_grad_(True))
                       for i, v in enumerate(train_views)]
        if not (config.intrinsics_learning_rate >= 0.0 and config.intrinsics_learning_rate < float("inf")):
            raise ValueError(f"intrinsics_learning_rate must be finite and >= 0, got {config.intrinsics_learning_rate}")
        self._intr = config.intrinsics_learning_rate > 0
        if self._intr and fused_step:
            raise ValueError("fused_step does not implement intrinsics refinement (intrinsics_learning_rate > 0)")
        # a view with lens distortion (CameraInfo.distortion) trains through the autograd loop alone
        if any(getattr(v[3], "distortion", None) is not None for v in train_views):
            for name, on in (("fused_step", fused_step), ("pose refinement (pose_learning_rate > 0)", self._pose),
                             ("intrinsics refinement (intrinsics_learning_rate > 0)", self._intr)):
                if on:
                    raise ValueError(f"{name} is not supported with a distorted view (CameraInfo.distortion)")
        # the trainable intrinsics corrections, one per camera_id: (log fx scale, log fy scale, cx / W, cy / H)
        self._intrinsics = {}
        if self._intr:
            for v in train_views:
                ci = v[3]
                if ci.camera_id not in self._intrinsics:
                    self._intrinsics[ci.camera_id] = torch.zeros(4, dtype=torch.float32, device=ci.camera_intrinsics.device,
                                                                 requires_grad=True)
        self._distortion = self._distortion_leaves(config, train_views)
        self._dist = config.distortion_learning_rate > 0
        # a view with a rolling shutter (CameraInfo.rolling_shutter) trains through the autograd loop alone
        if any(getattr(v[3], "rolling_shutter", None) is not None for v in train_views):
            for name, on in (("fused_step", fused_step), ("pose refinement (pose_learning_rate > 0)", self._pose),
                             ("intrinsics refinement (intrinsics_learning_rate > 0)", self._intr),
                             ("distortion refinement (distortion_learning_rate > 0)", self._dist)):
                if on:
                    raise ValueError(f"{name} is not supported with a rolling-shutter view (CameraInfo.rolling_shutter)")
        self._rolling_shutter = self._rolling_shutter_leaves(config, train_views)
        self._rs = config.rolling_shutter_learning_rate > 0
        self._mip = bool(config.mip_filter_3d)
        self._filter_3d = None
        if self._mip:
            v = config.mip_filter_variance
            if not (isinstance(v, (int, float)) and math.isfinite(v) and v >= 0):
                raise ValueError(f"mip_filter_variance must be finite and >= 0, got {v}")
            if not (isinstance(config.mip_filter_interval, int) and config.mip_filter_interval >= 1):
                raise ValueError(f"mip_filter_interval must be an int >= 1, got {config.mip_filter_interval!r}")
            for name, on in (("pose refinement (pose_learning_rate > 0)", self._pose),
                             ("intrinsics refinement (intrinsics_learning_rate > 0)", self._intr),
                             ("distortion refinement (distortion_learning_rate > 0)", config.distortion_learning_rate > 0),
                             ("motion refinement (rolling_shutter_learning_rate > 0)", self._rs)):
                if on:
                    raise ValueError(f"mip_filter_3d is not supported with {name}: the filter is computed from fixed "
                                     "training cameras")
            if any(getattr(getattr(v[3], "distortion", None), "model", None) == "fisheye" for v in train_views):
                raise ValueError("mip_filter_3d does not support fisheye training views: the filter's pinhole frustum test "
                                 "is wrong for them")
        self._appearance = config.appearance_grid is not None
        self._appearance_leaves = []
        self._appearance_tensor = None
        if self._appearance:
            shape = check_grid_shape(config.appearance_grid)
            for name in ("appearance_learning_rate", "appearance_tv_weight"):
                v = getattr(config, name)
                if not (v >= 0.0 and v < float("inf")):
                    raise ValueError(f"{name} must be finite and >= 0, got {v}")
            grids = identity_grids(len(train_views), shape, device=scene.point_cloud.device)
            if fused_step:  # updated in place by the fused step
                self._appearance_tensor = grids
            else:  # one leaf per view: an optimiser over them steps only the leaves that got a gradient
                self._appearance_leaves = [g.clone().requires_grad_(True) for g in grids]
        self._features = config.feature_loss != "none"
        if self._features:
            self._check_feature_config(config, scene, targets)
        if config.robust_loss is not None and not isinstance(config.robust_loss, RobustLossConfig):
            raise ValueError(f"robust_loss must be a RobustLossConfig, got {type(config.robust_loss).__name__}")
        # per-pixel weights of the image loss: the robust mask and / or a view's static loss_weight
        self._weighted = config.robust_loss is not None or any(tg.loss_weight is not None for tg in targets)
        self._robust_stats = None
        self.config = config
        self._need_depth = config.depth_loss_weight > 0
        self._need_alpha = config.mask_loss_weight > 0 or config.background != "black"
        self.supervised = self._need_depth or self._need_alpha
        self._background_generator = background_generator
        self._background = None
        if config.background == "white":
            self._background = torch.ones(3, dtype=torch.float32, device=scene.point_cloud.device)
        elif config.background == "random":
            self._background = torch.empty(3, dtype=torch.float32, device=scene.point_cloud.device)
        self.fused_step = fused_step
        if fused_step and config.loss_function_config.enable_regularization:
            raise ValueError("fused_step does not implement the optional scale regulariser (LossFunction.py:33-37)")
        self.fused_image_loss = fused_image_loss
        self.fused_adam = fused_adam
        self.scene = scene
        self.train_views = train_views
        maintained = GaussianPointAdaptiveController.GaussianPointAdaptiveControllerMaintainedParameters(
            pointcloud=scene.point_cloud, pointcloud_features=scene.point_cloud_features,
            point_invalid_mask=scene.point_invalid_mask, point_object_id=scene.point_object_id,
            point_extra_features=scene.point_extra_features if self._features else None)
        # one of the two: with MCMC there is no adaptive controller and no backward hook (no hook statistics)
        self.adaptive_controller = self.mcmc_controller = None
        if self._mcmc:
            self.mcmc_controller = GaussianPointMCMCController(config.mcmc_config, maintained, generator=generator)
        else:
            self.adaptive_controller = GaussianPointAdaptiveController(
                config=config.adaptive_controller_config, maintained_parameters=maintained, generator=generator,
                fused_update=fused_controller_update)
        factory = rasterisation_factory or GaussianPointCloudRasterisation
        # the differentiable outputs only when a term needs them: injected factories without them keep working
        extra = dict(**({"differentiable_depth": True} if self._need_depth else {}),
                     **({"differentiable_alpha": True} if self._need_alpha else {}),
                     **({"differentiable_pose": True} if self._pose else {}),
                     **({"differentiable_intrinsics": True} if self._intr else {}),
                     **({"differentiable_distortion": True} if self._dist else {}),
                     **({"differentiable_rolling_shutter": True} if self._rs else {}))
        self.rasterisation = factory(config=config.rasterisation_config,
                                     backward_valid_point_hook=None if self._mcmc else self.adaptive_controller.update,
                                     **extra)
        if self._mcmc and getattr(self.rasterisation, "gradient_exchange", None) is not None:
            raise ValueError('densification="mcmc" is not implemented for the view-parallel gradient exchange')
        if self._mip and getattr(self.rasterisation, "gradient_exchange", None) is not None:
            raise ValueError("mip_filter_3d is not implemented for the view-parallel gradient exchange")
        if self._weighted and getattr(self.rasterisation, "gradient_exchange", None) is not None:
            raise ValueError("robust_loss and per-view loss_weight targets are not implemented for the view-parallel "
                             "gradient exchange")
        self.loss_function = LossFunction(config=config.loss_function_config)
        self.history: List[dict] = []
        self._downsampled = {}
        self._view_generator = shuffle_generator
        self._view_order = None

    @staticmethod
    def _distortion_leaves(config, train_views: List[View]) -> dict:
        """The trainable lens coefficients, one float32 host leaf per camera_id with a lens ({} when lens refinement is off)."""
        rate = config.distortion_learning_rate
        if not (rate >= 0.0 and rate < float("inf")):
            raise ValueError(f"distortion_learning_rate must be finite and >= 0, got {rate}")
        if rate == 0:
            return {}
        lenses = {}
        for v in train_views:
            ci = v[3]
            lenses.setdefault(ci.camera_id, set()).add(getattr(ci, "distortion", None))
        for cid, found in lenses.items():
            if len(found) > 1:
                raise ValueError(f"the training views of camera_id {cid} have different lenses: {sorted(map(str, found))}")
        leaves = {cid: torch.tensor(lens.coefficients, dtype=torch.float32, requires_grad=True)
                  for cid, (lens,) in lenses.items() if lens is not None}
        if not leaves:
            raise ValueError("distortion_learning_rate > 0 needs a distorted training view (CameraInfo.distortion)")
        return leaves

    @staticmethod
    def _rolling_shutter_leaves(config, train_views: List[View]) -> dict:
        """The trainable motions, one float32 host leaf (6,) per rolling-shutter view, keyed by view index ({} when motion
        refinement is off)."""
        rate = config.rolling_shutter_learning_rate
        if not (rate >= 0.0 and rate < float("inf")):
            raise ValueError(f"rolling_shutter_learning_rate must be finite and >= 0, got {rate}")
        if rate == 0:
            return {}
        leaves = {i: torch.tensor(v[3].rolling_shutter.motion, dtype=torch.float32, requires_grad=True)
                  for i, v in enumerate(train_views) if getattr(v[3], "rolling_shutter", None) is not None}
        if not leaves:
            raise ValueError("rolling_shutter_learning_rate > 0 needs a rolling-shutter training view "
                             "(CameraInfo.rolling_shutter)")
        return leaves

    @staticmethod
    def _check_feature_config(config, scene: Scene, targets: List[SupervisionTargets]) -> None:
        if config.feature_loss not in FEATURE_LOSSES:
            raise ValueError(f"feature_loss must be one of {('none',) + FEATURE_LOSSES}, got {config.feature_loss!r}")
        w = config.feature_loss_weight
        if not (w > 0.0 and w < float("inf")):
            raise ValueError(f"feature_loss_weight must be finite and > 0 with a feature loss, got {w}")
        Fx = scene.point_extra_features
        if Fx is None:
            raise ValueError(f'feature_loss="{config.feature_loss}" needs Scene.point_extra_features')
        if Fx.dim() != 2 or Fx.shape[0] != scene.point_cloud.shape[0] or not 1 <= Fx.shape[1] <= 16:
            raise ValueError(f"point_extra_features must be (N, C) with 1 <= C <= 16, got {tuple(Fx.shape)}")
        C = int(Fx.shape[1])
        if config.feature_loss == "cross_entropy":
            if C < 2:
                raise ValueError(f'feature_loss="cross_entropy" needs C >= 2 channels, got {C}')
            if any(tg.labels is None for tg in targets):
                raise ValueError('feature_loss="cross_entropy" needs labels on every view')
            # one host read for all views: a label >= C is a class the features cannot express, not "no label"
            dev = targets[0].labels.device if targets else None
            top = int(torch.stack([tg.labels.max().to(dev, torch.int64) for tg in targets]).max()) if targets else -1
            if top >= C:
                raise ValueError(f"labels must be < C = {C} (negative = no label), got {top}")
        elif any(tg.features is None for tg in targets):
            raise ValueError('feature_loss="l2" needs a feature map on every view')
        elif any(tuple(tg.features.shape[-1:]) != (C,) for tg in targets):
            raise ValueError(f"the feature maps of the views must have C = {C} channels")

    def _input(self, q, t, camera_info, band):
        s = self.scene
        return GaussianPointCloudRasterisation.GaussianPointCloudRasterisationInput(
            point_cloud=s.point_cloud, point_cloud_features=s.point_cloud_features,
            point_object_id=s.point_object_id, point_invalid_mask=s.point_invalid_mask,
            camera_info=camera_info, q_pointcloud_camera=q, t_pointcloud_camera=t, color_max_sh_band=band)

    def _view(self, view_index: int, downsample_factor: int):
        """(image, q, t, camera, targets) of a view at the schedule's resolution; resized once per (view, factor)."""
        view = self.train_views[view_index]
        image_gt, _, _, camera_info = view[:4]
        q, t = self._poses[view_index]
        targets = view[4] if len(view) > 4 and view[4] is not None else SupervisionTargets()
        if downsample_factor > 1:
            # the reference resizes the full-resolution frame in every iteration (GaussianPointTrainer.py:146-148); the
            # result depends only on (view, factor), so it is computed once per pair (same tensors, ~10 launches less)
            key = (view_index, downsample_factor)
            if key not in self._downsampled:
                image_ds, camera_ds = downsample_image_and_camera_info(image_gt, camera_info, downsample_factor)
                self._downsampled[key] = (image_ds, camera_ds, downsample_targets(targets, camera_info, downsample_factor)
                                          if self.supervised or self._features or self._weighted else targets)
            image_gt, camera_info, targets = self._downsampled[key]
        return image_gt, q, t, camera_info, targets

    def _intrinsics_of(self, view_index: int, downsample_factor: int) -> torch.Tensor:
        """The K of a view as trained, built by torch ops (differentiable in its camera's correction): the view's own
        full-resolution K with fx, fy scaled by exp(log-scale) and cx, cy shifted by offset * (W, H), then fx, fy, cx, cy
        divided by the downsample factor as ``downsample_image_and_camera_info`` does."""
        ci = self.train_views[view_index][3]
        K = ci.camera_intrinsics
        corr = self._intrinsics[ci.camera_id]
        rows, cols = torch.tensor([0, 1], device=K.device), torch.tensor([2, 2], device=K.device)
        size = torch.tensor([float(ci.camera_width), float(ci.camera_height)], dtype=K.dtype, device=K.device)
        scale = torch.ones_like(K).index_put((rows, rows), torch.exp(corr[:2]))
        shift = torch.zeros_like(K).index_put((rows, cols), corr[2:] * size)
        K = K * scale + shift
        if downsample_factor > 1:
            div = torch.ones_like(K).index_put((torch.tensor([0, 1, 0, 1], device=K.device),
                                                torch.tensor([0, 1, 2, 2], device=K.device)),
                                               torch.tensor(float(downsample_factor), dtype=K.dtype, device=K.device))
            K = K / div
        return K

    def _update_filter_3d(self) -> None:
        """The 3D filter of the current rows from the full-resolution training views (``mip_filter.compute_filter_3d``)."""
        views = [(q, t, v[3]) for (q, t), v in zip(self._poses, self.train_views)]
        self._filter_3d = compute_filter_3d(self.scene.point_cloud, self.scene.point_invalid_mask, self.scene.point_object_id,
                                            views, self.config.rasterisation_config.near_plane, self.config.mip_filter_variance)

    def _after_refinement(self, iteration: int) -> None:
        """Recomputes the 3D filter after a refinement that may have moved rows (densification, MCMC relocation and growth)
        and every ``mip_filter_interval`` iterations."""
        if not self._mip:
            return
        if self._mcmc:
            c = self.mcmc_controller
            refined = c.config.refine_start <= c.iteration_counter < c.config.refine_stop and \
                c.iteration_counter % c.config.refine_every == 0
        else:
            c = self.adaptive_controller
            refined = c.iteration_counter >= c.config.num_iterations_warm_up and \
                c.iteration_counter % c.config.num_iterations_densify == 0
        if refined or (iteration + 1) % self.config.mip_filter_interval == 0:
            self._update_filter_3d()

    def _filter_kw(self) -> dict:
        return {"point_filter_3d": self._filter_3d} if self._mip else {}

    def filter_3d(self) -> Optional[torch.Tensor]:
        """The (N,) 3D filter the latest iteration rendered with (a detached copy; None without ``mip_filter_3d``).
        ``GaussianPointCloudScene.to_ply(path, filter_3d=...)`` bakes it into an export."""
        return None if self._filter_3d is None else self._filter_3d.detach().clone()

    def _next_background(self) -> Optional[torch.Tensor]:
        """The background of this iteration: None (black), white, or a fresh colour drawn on the device."""
        if self.config.background == "random":
            torch.rand(3, generator=self._background_generator, out=self._background)
        return self._background

    def _supervised_history(self, entry: dict, mask_term, depth_term) -> dict:
        if self.config.mask_loss_weight > 0:
            entry["mask_loss"] = float(mask_term)
        if self.config.depth_loss_weight > 0:
            entry["depth_loss"] = float(depth_term)
        return entry

    def _train_fused(self, log_interval: int = 0):
        """The loop of ``train`` with the whole iteration enqueued by ONE library call (``fused_step.FusedTrainStep``):
        no autograd graph, no host wait, the controller's accumulators updated inside the backward kernel."""
        from .fused_step import FusedTrainStep
        cfg = self.config
        step = FusedTrainStep(self.scene, cfg.rasterisation_config, cfg.loss_function_config.lambda_value,
                              controller=self.adaptive_controller, depth_weight=cfg.depth_loss_weight,
                              mask_weight=cfg.mask_loss_weight, mcmc=cfg.mcmc_config if self._mcmc else None,
                              robust=cfg.robust_loss,
                              **(dict(extra_features=self.scene.point_extra_features, feature_loss=cfg.feature_loss,
                                      feature_weight=cfg.feature_loss_weight,
                                      extra_feature_learning_rate=cfg.extra_feature_learning_rate) if self._features else {}),
                              **(dict(appearance_grids=self._appearance_tensor,
                                      appearance_learning_rate=cfg.appearance_learning_rate,
                                      appearance_tv_weight=cfg.appearance_tv_weight) if self._appearance else {}))
        self.fused_train_step = step
        position_lr = cfg.position_learning_rate
        downsample_factor = cfg.initial_downsample_factor
        if self._mip:
            self._update_filter_3d()
        for iteration in range(cfg.num_iterations):
            if iteration % cfg.half_downsample_factor_interval == 0 and iteration > 0 and downsample_factor > 1:
                downsample_factor //= 2
            view_index = self._next_view_index(iteration)
            image_gt, q, t, camera_info, targets = self._view(view_index, downsample_factor)
            band = iteration // cfg.increase_color_max_sh_band_interval
            app_kw = {"appearance_view": view_index} if self._appearance else {}
            if self._mcmc:
                app_kw["mcmc_num_valid"] = self.mcmc_controller.num_valid
            if self._mip:
                app_kw["filter_3d"] = self._filter_3d
            if cfg.robust_loss is not None:
                app_kw["robust_active"] = iteration >= cfg.robust_loss.start_iteration
            if self.supervised or self._features or self._weighted:
                step.run(image_gt, q, t, camera_info, band, cfg.feature_learning_rate, position_lr, targets=targets,
                         background=self._next_background(), **app_kw)
            else:
                step.run(image_gt, q, t, camera_info, band, cfg.feature_learning_rate, position_lr, **app_kw)
            if iteration % cfg.position_learning_rate_decay_interval == 0:  # ExponentialLR.step() after the optimiser step
                position_lr *= cfg.position_learning_rate_decay_rate
            if self._mcmc:
                self.mcmc_controller.refinement(step.moments)
            else:
                self.adaptive_controller.after_fused_update(step.hook_input)
                self.adaptive_controller.refinement()
            self._after_refinement(iteration)
            if log_interval and iteration % log_interval == 0:
                losses = step.loss.tolist()
                entry = dict(iteration=iteration, loss=losses[0], l1=losses[1],
                             psnr=psnr(step.image.detach().clamp(0, 1).permute(2, 0, 1), image_gt),
                             num_valid_points=int((self.scene.point_invalid_mask == 0).sum()))
                if self.supervised:
                    total, mask_term, depth_term = step.supervision_loss.tolist()
                    entry["loss"] = total
                    self._supervised_history(entry, mask_term, depth_term)
                if self._features:
                    entry["feature_loss"] = float(step.feature_loss[0])
                    entry["loss"] += entry["feature_loss"]
                if self._appearance:
                    entry["appearance_tv"] = float(step.appearance_tv[0])
                    entry["loss"] += entry["appearance_tv"]
                if self._mcmc:
                    entry["mcmc_opacity_reg"], entry["mcmc_scale_reg"] = step.mcmc_terms.tolist()
                    entry["loss"] += entry["mcmc_opacity_reg"] + entry["mcmc_scale_reg"]
                if self._weighted:
                    entry["robust_inlier_fraction"] = float(step.robust_stats[0]) if step.loss_weight is not None else 1.0
                self.history.append(entry)
        return self.history

    def _next_view_index(self, iteration: int) -> int:
        """A fresh random permutation of the views every epoch (the reference draws them from a DataLoader with shuffle=True,
        GaussianPointTrainer.py:120-124), seeded from the injected generator; without a generator: the fixed order
        ``iteration % len(views)`` (deterministic tests and golden trajectories)."""
        n = len(self.train_views)
        if self._view_generator is None:
            return iteration % n
        k = iteration % n
        if k == 0 or self._view_order is None:
            self._view_order = torch.randperm(n, generator=self._view_generator).tolist()
        return self._view_order[k]

    def train(self, log_interval: int = 0):
        if self.fused_step:
            return self._train_fused(log_interval)
        cfg = self.config
        if self.fused_adam:
            from .optim import FusedAdam as Adam
        else:
            Adam = torch.optim.Adam
        optimizer = Adam([self.scene.point_cloud_features], lr=cfg.feature_learning_rate, betas=(0.9, 0.999))
        position_optimizer = Adam([self.scene.point_cloud], lr=cfg.position_learning_rate, betas=(0.9, 0.999))
        extra_optimizer = Adam([self.scene.point_extra_features], lr=cfg.extra_feature_learning_rate,
                               betas=(0.9, 0.999)) if self._features else None
        pose_optimizer = Adam([x for q, t in self._poses[1:] for x in (q, t)], lr=cfg.pose_learning_rate,
                              betas=(0.9, 0.999)) if self._pose and len(self._poses) > 1 else None
        intrinsics_optimizer = Adam(list(self._intrinsics.values()), lr=cfg.intrinsics_learning_rate,
                                    betas=(0.9, 0.999)) if self._intr else None
        # host tensors: torch's Adam whatever fused_adam says
        distortion_optimizer = torch.optim.Adam(list(self._distortion.values()), lr=cfg.distortion_learning_rate,
                                                betas=(0.9, 0.999)) if self._dist else None
        rolling_shutter_optimizer = torch.optim.Adam(list(self._rolling_shutter.values()),
                                                     lr=cfg.rolling_shutter_learning_rate, betas=(0.9, 0.999)) \
            if self._rs else None
        appearance_optimizer = Adam(self._appearance_leaves, lr=cfg.appearance_learning_rate, betas=(0.9, 0.999)) \
            if self._appearance else None
        scheduler = torch.optim.lr_scheduler.ExponentialLR(position_optimizer, gamma=cfg.position_learning_rate_decay_rate)
        downsample_factor = cfg.initial_downsample_factor
        if self._mip:
            self._update_filter_3d()
        for iteration in range(cfg.num_iterations):
            if iteration % cfg.half_downsample_factor_interval == 0 and iteration > 0 and downsample_factor > 1:
                downsample_factor //= 2
            optimizer.zero_grad()
            position_optimizer.zero_grad()
            if extra_optimizer is not None:
                extra_optimizer.zero_grad()
            if pose_optimizer is not None:
                pose_optimizer.zero_grad()
            if intrinsics_optimizer is not None:
                intrinsics_optimizer.zero_grad()
            if distortion_optimizer is not None:
                distortion_optimizer.zero_grad()
            if rolling_shutter_optimizer is not None:
                rolling_shutter_optimizer.zero_grad()
            if appearance_optimizer is not None:
                appearance_optimizer.zero_grad()
            view_index = self._next_view_index(iteration)
            image_gt, q, t, camera_info, targets = self._view(view_index, downsample_factor)
            if self._intr:  # built every iteration: the cached downsampled camera must not freeze K
                camera_info = CameraInfo(camera_intrinsics=self._intrinsics_of(view_index, downsample_factor),
                                         camera_height=camera_info.camera_height, camera_width=camera_info.camera_width,
                                         camera_id=camera_info.camera_id)
            lens_kw = self._filter_kw()
            if self._dist and camera_info.distortion is not None:  # the lens as trained, the leaf as the autograd input
                leaf = self._distortion[camera_info.camera_id]
                camera_info = CameraInfo(camera_intrinsics=camera_info.camera_intrinsics,
                                         camera_height=camera_info.camera_height, camera_width=camera_info.camera_width,
                                         camera_id=camera_info.camera_id,
                                         distortion=LensDistortion(camera_info.distortion.model, leaf.detach().tolist()))
                lens_kw = {"lens_coefficients": leaf}
            if self._rs and view_index in self._rolling_shutter:  # the motion as trained, the leaf as the autograd input
                leaf = self._rolling_shutter[view_index]
                values = leaf.detach().tolist()
                camera_info = CameraInfo(camera_intrinsics=camera_info.camera_intrinsics,
                                         camera_height=camera_info.camera_height, camera_width=camera_info.camera_width,
                                         camera_id=camera_info.camera_id, distortion=camera_info.distortion,
                                         rolling_shutter=RollingShutter(values[:3], values[3:]))
                lens_kw = {"rolling_shutter_motion": leaf}
            band = iteration // cfg.increase_color_max_sh_band_interval
            if self.supervised or self._features or self._appearance or self._weighted:
                robust_active = cfg.robust_loss is not None and iteration >= cfg.robust_loss.start_iteration
                loss, l1_loss, mask_term, depth_term, feature_term, appearance_tv, image_pred = self._supervised_loss(
                    q, t, camera_info, band, image_gt, targets, lens_kw, view_index, robust_active)
            elif self.fused_image_loss:
                image_pred, _, _ = self.rasterisation(self._input(q, t, camera_info, band), **lens_kw)
                loss, l1_loss, ssim_loss = self.loss_function.forward_rasterized(
                    image_pred, image_gt, point_invalid_mask=self.scene.point_invalid_mask,
                    pointcloud_features=self.scene.point_cloud_features)
                image_pred = image_pred.detach().clamp(0, 1).permute(2, 0, 1) if log_interval else image_pred
            else:
                image_pred, _, _ = self.rasterisation(self._input(q, t, camera_info, band), **lens_kw)
                image_pred = torch.clamp(image_pred, min=0, max=1).permute(2, 0, 1)
                loss, l1_loss, ssim_loss = self.loss_function(
                    image_pred, image_gt, point_invalid_mask=self.scene.point_invalid_mask,
                    pointcloud_features=self.scene.point_cloud_features)
            if self._mcmc:
                mc = cfg.mcmc_config
                mcmc_terms = mcmc_regulariser(self.scene.point_cloud_features, self.scene.point_invalid_mask, mc.opacity_reg,
                                              mc.scale_reg, num_valid=self.mcmc_controller.num_valid)
                loss = loss + mcmc_terms.sum()
            loss.backward()
            optimizer.step()
            position_optimizer.step()
            if extra_optimizer is not None:
                extra_optimizer.step()
            if pose_optimizer is not None:
                pose_optimizer.step()
                with torch.no_grad():
                    for q_v, _ in self._poses[1:]:
                        q_v.div_(q_v.norm(dim=-1, keepdim=True))
            if intrinsics_optimizer is not None:
                intrinsics_optimizer.step()
            if distortion_optimizer is not None:
                distortion_optimizer.step()
            if rolling_shutter_optimizer is not None:
                rolling_shutter_optimizer.step()
            if appearance_optimizer is not None:
                appearance_optimizer.step()
            if self._mcmc:  # the noise of iteration t at the position learning rate its optimiser step used
                add_position_noise(self.scene.point_cloud, self.scene.point_cloud_features, self.scene.point_invalid_mask,
                                   mc.noise_lr * position_optimizer.param_groups[0]["lr"], mc.seed, iteration, GATE_K,
                                   mc.min_opacity)
            if iteration % cfg.position_learning_rate_decay_interval == 0:
                scheduler.step()
            if self._mcmc:
                self.mcmc_controller.refinement(MCMCMoments.of_optimizers(optimizer, position_optimizer, extra_optimizer))
            else:
                self.adaptive_controller.refinement()
            self._after_refinement(iteration)
            if log_interval and iteration % log_interval == 0:
                entry = dict(iteration=iteration, loss=float(loss.detach()), l1=float(l1_loss.detach()),
                             psnr=psnr(image_pred.detach(), image_gt),
                             num_valid_points=int((self.scene.point_invalid_mask == 0).sum()))
                if self.supervised:
                    self._supervised_history(entry, mask_term.detach(), depth_term.detach())
                if self._features:
                    entry["feature_loss"] = float(feature_term.detach())
                if self._appearance:
                    entry["appearance_tv"] = float(appearance_tv.detach())
                if self._mcmc:
                    entry["mcmc_opacity_reg"], entry["mcmc_scale_reg"] = mcmc_terms.detach().tolist()
                if self._weighted:
                    entry["robust_inlier_fraction"] = float(self._robust_stats[0]) if self._robust_stats is not None else 1.0
                self.history.append(entry)
        return self.history

    def _supervised_loss(self, q, t, camera_info, band, image_gt, targets, lens_kw=None, view_index=None,
                         robust_active=False):
        """Forward with the differentiable outputs the terms need, then ``loss.supervision_loss`` with this trainer's image
        loss (the torch one, or the fused kernels with ``fused_image_loss``; the scale regulariser if enabled), plus
        ``loss.feature_loss`` on the rendered feature map with a feature loss.  Returns (total, L1, mask term, depth term,
        feature term, the weighted TV term of the appearance grid, the raw image as (3, H, W) for the PSNR log).
        ``lens_kw``: the operator's ``lens_coefficients`` argument with lens refinement.  With appearance grids the image
        loss reads the image (after the background composite) sliced through the grid of ``view_index``.  With loss weights
        (the view's ``targets.loss_weight``, and the robust mask when ``robust_active``) the image loss reads the composite
        ``loss.robust_composite`` of that image under ``loss.robust_weight``."""
        cfg = self.config
        lens_kw = lens_kw or {}
        if self._features:
            outs = self.rasterisation(self._input(q, t, camera_info, band), point_extra_features=self.scene.point_extra_features,
                                      **lens_kw)
        else:
            outs = self.rasterisation(self._input(q, t, camera_info, band), **lens_kw)
        image_pred, depth = outs[0], outs[1]
        alpha = outs[3] if self._need_alpha else None
        regulariser = dict(point_invalid_mask=self.scene.point_invalid_mask, pointcloud_features=self.scene.point_cloud_features)
        if self.fused_image_loss:
            image_loss = lambda pred, gt: self.loss_function.forward_rasterized(pred, gt, **regulariser)  # noqa: E731
        else:
            image_loss = lambda pred, gt: self.loss_function(  # noqa: E731
                torch.clamp(pred, min=0, max=1).permute(2, 0, 1), gt, **regulariser)
        self._robust_stats = None
        static_w = targets.loss_weight if targets is not None else None
        if robust_active or static_w is not None:
            weighted_image_loss = image_loss
            robust_cfg = cfg.robust_loss if robust_active else None

            def image_loss(pred, gt):
                w, self._robust_stats = robust_weight(pred.detach(), gt, static_w, robust_cfg)
                return weighted_image_loss(robust_composite(pred, gt, w), gt)
        appearance_tv = None
        if self._appearance:
            grid = self._appearance_leaves[view_index]
            raw_image_loss = image_loss
            image_loss = lambda pred, gt: raw_image_loss(apply_bilateral_grid(pred, grid), gt)  # noqa: E731
            appearance_tv = cfg.appearance_tv_weight * bilateral_grid_tv(grid)
        total, l1, _, mask_term, depth_term = supervision_loss(
            image_pred, depth, alpha, image_gt, targets, self._next_background(), cfg.loss_function_config.lambda_value,
            cfg.depth_loss_weight, cfg.mask_loss_weight, image_loss=image_loss)
        feature_term = None
        if self._features:
            feature_term = feature_loss(outs[-1], targets, cfg.feature_loss, cfg.feature_loss_weight)
            total = total + feature_term
        if appearance_tv is not None:
            total = total + appearance_tv
        return (total, l1, mask_term, depth_term, feature_term, appearance_tv,
                image_pred.detach().clamp(0, 1).permute(2, 0, 1))

    def appearance_grids(self) -> Optional[torch.Tensor]:
        """The (V, 12, Gz, Gy, Gx) appearance grids of the training views as trained (a detached copy; None without
        appearance compensation)."""
        if not self._appearance:
            return None
        if self._appearance_tensor is not None:
            return self._appearance_tensor.detach().clone()
        return torch.stack([g.detach() for g in self._appearance_leaves]).clone()

    def refined_poses(self) -> List[Tuple[torch.Tensor, torch.Tensor]]:
        """(q, t) of every training view as trained (detached copies; the views' own poses without pose refinement)."""
        return [(q.detach().clone(), t.detach().clone()) for q, t in self._poses]

    def refined_intrinsics(self) -> List[torch.Tensor]:
        """The full-resolution (3, 3) K of every training view as trained (detached copies; the views' own K without
        intrinsics refinement)."""
        if not self._intr:
            return [v[3].camera_intrinsics.detach().clone() for v in self.train_views]
        with torch.no_grad():
            return [self._intrinsics_of(i, 1).clone() for i in range(len(self.train_views))]

    def refined_distortion(self) -> List[Optional[LensDistortion]]:
        """The lens of every training view as trained (None for a view without one; the views' own lenses without lens
        refinement)."""
        out = []
        for v in self.train_views:
            ci = v[3]
            lens = getattr(ci, "distortion", None)
            if lens is not None and ci.camera_id in self._distortion:
                lens = LensDistortion(lens.model, self._distortion[ci.camera_id].detach().tolist())
            out.append(lens)
        return out

    def refined_rolling_shutter(self) -> List[Optional[RollingShutter]]:
        """The rolling shutter of every training view as trained (None for a view without one; the views' own motions
        without motion refinement)."""
        out = []
        for i, v in enumerate(self.train_views):
            rs = getattr(v[3], "rolling_shutter", None)
            if rs is not None and i in self._rolling_shutter:
                values = self._rolling_shutter[i].detach().tolist()
                rs = RollingShutter(values[:3], values[3:])
            out.append(rs)
        return out

    @torch.no_grad()
    def validation(self, views: Optional[List[View]] = None) -> float:
        """Mean PSNR over the views at full resolution (GaussianPointTrainer.py:334-415 without the logging)."""
        views = views if views is not None else self.train_views
        if self._mip and self._filter_3d is None:
            self._update_filter_3d()
        total = 0.0
        for view in views:
            image_gt, q, t, camera_info = view[:4]
            outs = self.rasterisation(self._input(q, t, camera_info, 3), **self._filter_kw())
            image_pred = outs[0]
            if self.config.background != "black":
                # white: the prediction on white and the ground truth composited by its mask; random: both on black
                bg = 1.0 if self.config.background == "white" else 0.0
                if bg:
                    image_pred = image_pred + (1 - outs[3])[..., None] * bg
                mask = view[4].mask if len(view) > 4 and view[4] is not None else None
                if mask is not None:
                    image_gt = image_gt * mask[None] + (1 - mask)[None] * bg
            total += psnr(image_pred.permute(2, 0, 1), image_gt)
        return total / max(len(views), 1)
