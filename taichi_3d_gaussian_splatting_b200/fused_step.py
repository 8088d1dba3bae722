"""``FusedTrainStep``: one training iteration of the reference loop (``GaussianPointTrainer.py:138-180``) as ONE call into
``libgsb200.so`` (``gsb200_train_step``): forward, clamp + L1 + D-SSIM loss and its gradient, backward with the densification
controller's accumulators updated in the epilogue of the per-point kernel, Adam on the features and on the positions --
about 15 kernels enqueued back to back with no host wait, no autograd graph and no per-iteration allocation.  The Python
trainer around it (``trainer.GaussianPointCloudTrainer(..., fused_step=True)``) only picks the view, computes the two
learning rates and runs the controller's ``refinement`` every ``num_iterations_densify`` iterations.

What the host does NOT know any more: the number of in-camera points M and of (tile, splat) pairs K of a frame (the operator
waits for them once per frame; here nothing waits).  The accumulator buffer therefore has N rows, and a frame that needs more
pairs than the key capacity turns itself into a no-op ON THE DEVICE (overflow counter checked by the accumulator update and
both Adam kernels); the host reads the counters of iteration i while it prepares iteration i+1, grows the capacity and counts
the skipped iteration in ``num_skipped_steps``.  CUDA only; there is no CPU path.

Optional supervision terms (``depth_weight``, ``mask_weight``, ``run(..., targets=, background=)``): a masked-L1 depth loss,
an L1 mask loss on the accumulated alpha and training on a background colour, in the same one call
(``gsb200_train_step_aux``; ``loss.supervision_loss`` states the loss in torch).

Optional feature term (``extra_features``, ``feature_loss``, ``run(..., targets=SupervisionTargets(labels=... | features=...))``):
per-Gaussian feature vectors F (N, C) rendered alongside the image, a cross-entropy or l2 loss on the rendered (H, W, C) map
and an Adam step on F, in the same one call (``gsb200_train_step_ext``; ``loss.feature_loss`` states the loss in torch).

Optional appearance grids (``appearance_grids``, ``run(..., appearance_view=i)``): one bilateral grid per training view
(``appearance.apply_bilateral_grid``) slices the image the image loss reads, with a TV prior and an Adam step on the visited
view's grid, in the same one call (``gsb200_train_step_appearance``).  Each view has its own Adam moments and its own step
count, as torch's Adam gives one parameter per view that only steps when it has a gradient.

Optional MCMC densification (``mcmc=MCMCConfig``, ``run(..., mcmc_num_valid=n_v)``): the opacity and scale regularisers are
added to the feature gradient between the backward and the Adam steps and the covariance-shaped position noise after them, in
the same one call (``gsb200_train_step_mcmc``; ``loss.mcmc_regulariser`` and ``mcmc.add_position_noise`` state them in torch).
The refinements stay on the host (``mcmc.GaussianPointMCMCController.refinement(step.moments)``).
"""
import ctypes
import warnings
from types import SimpleNamespace
from typing import Optional

import torch

from . import _lib
from .GaussianPointCloudRasterisation import Frame, GaussianPointCloudRasterisation, _ptr
from .loss import FEATURE_LOSSES, SupervisionTargets
from .mcmc import GATE_K, MCMCMoments

__all__ = ["FusedTrainStep", "SupervisionTargets"]


class FusedTrainStep:
    def __init__(self, scene, rasterisation_config, lambda_value: float = 0.2, controller=None, betas=(0.9, 0.999),
                 eps: float = 1e-8, key_capacity: Optional[int] = None, depth_weight: float = 0.0,
                 mask_weight: float = 0.0, extra_features: Optional[torch.Tensor] = None, feature_loss: Optional[str] = None,
                 feature_weight: float = 1.0, extra_feature_learning_rate: float = 1e-2,
                 appearance_grids: Optional[torch.Tensor] = None, appearance_learning_rate: float = 2e-3,
                 appearance_tv_weight: float = 10.0, mcmc=None):
        """``scene``: object with ``point_cloud`` (N,3), ``point_cloud_features`` (N,56), ``point_invalid_mask``,
        ``point_object_id`` (CUDA, contiguous; updated in place).  ``controller``: a ``GaussianPointAdaptiveController`` whose
        six accumulators are updated by the backward epilogue (or ``None``).  ``depth_weight`` / ``mask_weight``: weights of
        the depth and mask terms (``loss.supervision_loss``); they need the matching target in ``run(targets=...)``.
        ``extra_features``: (N, C) float32 per-Gaussian feature vectors (CUDA, contiguous, 1 <= C <= 16; updated in place by
        their own Adam at ``extra_feature_learning_rate``), trained with ``feature_loss`` ("cross_entropy": needs
        ``targets.labels`` and C >= 2; "l2": needs ``targets.features``) weighted by ``feature_weight``
        (``loss.feature_loss``).  ``appearance_grids``: (V, 12, Gz, Gy, Gx) float32 per-view bilateral grids (CUDA,
        contiguous; updated in place), trained at ``appearance_learning_rate`` with the TV weight ``appearance_tv_weight``;
        ``run`` then needs ``appearance_view``.  ``mcmc``: an ``mcmc.MCMCConfig``; ``run`` then needs ``mcmc_num_valid``."""
        for name, w in (("depth_weight", depth_weight), ("mask_weight", mask_weight)):
            if not (w >= 0.0 and w < float("inf")):
                raise ValueError(f"{name} must be finite and >= 0, got {w}")
        self.depth_weight, self.mask_weight = float(depth_weight), float(mask_weight)
        self.extra_features = extra_features
        self.feature_loss_kind = feature_loss
        self.feature_weight = float(feature_weight)
        self.extra_feature_learning_rate = float(extra_feature_learning_rate)
        if (extra_features is None) != (feature_loss is None):
            raise ValueError("extra_features and feature_loss must be given together")
        self.scene = scene
        self.config = rasterisation_config
        self.lambda_value = float(lambda_value)
        self.controller = controller
        self.betas, self.eps = betas, float(eps)
        pc = scene.point_cloud
        if not pc.is_cuda:
            raise RuntimeError("FusedTrainStep needs CUDA tensors: there is no CPU path")
        self.device = pc.device
        self.N = pc.shape[0]
        self.key_capacity = int(key_capacity) if key_capacity else max(1 << 20, 8 * self.N)
        self.step_count = 0
        self.num_skipped_steps = 0
        self._lib = _lib.load()
        dev, N = self.device, self.N
        z = lambda *shape: torch.zeros(shape, dtype=torch.float32, device=dev)  # noqa: E731
        self.feature_exp_avg, self.feature_exp_avg_sq = z(N, 56), z(N, 56)
        self.position_exp_avg, self.position_exp_avg_sq = z(N, 3), z(N, 3)
        self.accum = torch.empty((max(N, 1), 12), dtype=torch.float32, device=dev)
        off = (3 * N + 3) // 4 * 4
        self._flat = z(off + 56 * N)
        self.grad_pointcloud = self._flat[:3 * N].view(N, 3)
        self.grad_pointcloud_features = self._flat[off:off + 56 * N].view(N, 56)
        self.loss = z(3)  # {loss, L1, 1 - SSIM} of the latest iteration (device); with supervision terms: of the image loss
        self.supervision_loss = z(3)  # {total, mask term, depth term} of the latest supervised iteration (device)
        self.feature_loss = z(2)  # {feature term, n_supervised} of the latest iteration with features (device)
        if extra_features is not None:
            self.C = self._check_extra_features(extra_features)
            if feature_loss not in FEATURE_LOSSES:
                raise ValueError(f"feature_loss must be one of {FEATURE_LOSSES}, got {feature_loss!r}")
            if feature_loss == "cross_entropy" and self.C < 2:
                raise ValueError(f'feature_loss "cross_entropy" needs C >= 2 channels, got {self.C}')
            if not (self.feature_weight > 0.0 and self.feature_weight < float("inf")):
                raise ValueError(f"feature_weight must be finite and > 0, got {feature_weight}")
            self.extra_feature_exp_avg, self.extra_feature_exp_avg_sq = z(N, self.C), z(N, self.C)
            self.grad_extra_features = z(N, self.C)
        self.appearance_grids = appearance_grids
        if appearance_grids is not None:
            self._check_appearance(appearance_grids, appearance_learning_rate, appearance_tv_weight)
            self.appearance_learning_rate = float(appearance_learning_rate)
            self.appearance_tv_weight = float(appearance_tv_weight)
            V = appearance_grids.shape[0]
            self.appearance_exp_avg = torch.zeros_like(appearance_grids)
            self.appearance_exp_avg_sq = torch.zeros_like(appearance_grids)
            self.appearance_steps = [0] * V  # each view's own Adam step count
            self.grad_appearance_grid = torch.zeros_like(appearance_grids[0])
        self.appearance_tv = z(1)  # {tv_weight * tv(G)} of the latest iteration with appearance (device)
        self.mcmc = mcmc.check() if mcmc is not None else None
        self.mcmc_terms = z(2)  # {opacity term, scale term} of the latest iteration with MCMC (device)
        if mcmc is not None:
            self._mcmc_temp = torch.zeros(int(self._lib.gsb200_mcmc_temp_bytes()), dtype=torch.uint8, device=dev)
        self._res = {}
        self._pinned = [torch.zeros(4, dtype=torch.int64).pin_memory() for _ in range(2)]
        self._events = [torch.cuda.Event() for _ in range(2)]
        for e in self._events:
            e.record()
        self._pending = [False, False]
        self._last = None

    def _check_extra_features(self, F) -> int:
        if not isinstance(F, torch.Tensor) or F.dim() != 2 or F.shape[0] != self.N or not 1 <= F.shape[1] <= 16:
            raise ValueError(f"extra_features must be an (N, C) tensor with N = {self.N} and 1 <= C <= 16, got "
                             f"{tuple(F.shape) if isinstance(F, torch.Tensor) else type(F).__name__}")
        if F.dtype != torch.float32 or F.device != self.device or not F.is_contiguous() or F.data_ptr() % 16:
            raise ValueError(f"extra_features must be a contiguous, 16-byte aligned float32 tensor on {self.device}")
        return int(F.shape[1])

    def _check_appearance(self, G, lr, tv_weight):
        from .appearance import check_grid_shape
        if not isinstance(G, torch.Tensor) or G.dim() != 5 or G.shape[0] < 1 or G.shape[1] != 12:
            raise ValueError(f"appearance_grids must be a (V, 12, Gz, Gy, Gx) tensor, got "
                             f"{tuple(G.shape) if isinstance(G, torch.Tensor) else type(G).__name__}")
        check_grid_shape((G.shape[4], G.shape[3], G.shape[2]))
        if G.dtype != torch.float32 or G.device != self.device or not G.is_contiguous() or G.data_ptr() % 16:
            raise ValueError(f"appearance_grids must be a contiguous, 16-byte aligned float32 tensor on {self.device}")
        for name, v in (("appearance_learning_rate", lr), ("appearance_tv_weight", tv_weight)):
            if not (v >= 0.0 and v < float("inf")):
                raise ValueError(f"{name} must be finite and >= 0, got {v}")

    # ------------------------------------------------------------------ per-resolution buffers
    def _buffers(self, H, W, n_obj):
        key = (H, W, n_obj, self.key_capacity)
        b = self._res.get(key)
        if b is None:
            cfg, dev = self.config, self.device
            layout = _lib.workspace_layout(self.N, n_obj, self.key_capacity, H, W, cfg.far_plane, cfg.depth_to_sort_key_scale, 0)
            e = lambda shape, dt=torch.float32: torch.empty(shape, dtype=dt, device=dev)  # noqa: E731
            temp_bytes = int(self._lib.gsb200_image_loss_temp_bytes(H, W))
            sup_bytes = int(self._lib.gsb200_supervision_temp_bytes(H, W))
            b = SimpleNamespace(layout=layout, ws=e((layout.total_bytes,), torch.uint8), image=e((H, W, 3)), depth=e((H, W)),
                                acc_alpha=e((H, W)), last_effective=e((H, W), torch.int32), count=e((H, W), torch.int32),
                                grad_image=e((H, W, 3)), mag_image=e((H, W, 2)),
                                loss_temp=torch.zeros((temp_bytes + 15) // 16 * 16, dtype=torch.uint8, device=dev),
                                temp_bytes=temp_bytes, grad_depth=e((H, W)), grad_alpha=e((H, W)),
                                sup_temp=torch.zeros((sup_bytes + 15) // 16 * 16, dtype=torch.uint8, device=dev),
                                sup_bytes=sup_bytes)
            if self.extra_features is not None:
                feat_bytes = int(self._lib.gsb200_feature_loss_temp_bytes(H, W))
                b.feature_map, b.grad_feature_map = e((H, W, self.C)), e((H, W, self.C))
                b.feat_temp = torch.zeros((feat_bytes + 15) // 16 * 16, dtype=torch.uint8, device=dev)
                b.feat_bytes = feat_bytes
            if self.appearance_grids is not None:
                gz, gy, gx = self.appearance_grids.shape[2:]
                app_bytes = int(self._lib.gsb200_bilateral_grid_temp_bytes(H, W, gx, gy, gz))
                b.sliced_image = e((H, W, 3))
                b.app_temp = torch.zeros((app_bytes + 15) // 16 * 16, dtype=torch.uint8, device=dev)
                b.app_bytes = app_bytes
            self._res[key] = b
        return b

    def _check_previous(self):
        """Counters of the iteration before the latest one (their copy finished long ago): overflow -> grow and count."""
        slot = self.step_count % 2
        if not self._pending[slot]:
            return
        self._events[slot].synchronize()
        self._pending[slot] = False
        if int(self._pinned[slot][2]) != 0:
            needed = int(self._pinned[slot][1])
            self.key_capacity = int(needed * 1.25) + 4096
            self.num_skipped_steps += 1
            warnings.warn(f"FusedTrainStep: a frame needed {needed} (tile, splat) pairs; that iteration was a no-op on the device, "
                          f"the key capacity is now {self.key_capacity}")

    # ------------------------------------------------------------------ one iteration
    def run(self, image_gt: torch.Tensor, q_pointcloud_camera: torch.Tensor, t_pointcloud_camera: torch.Tensor, camera_info,
            color_max_sh_band: int, feature_learning_rate: float, position_learning_rate: float,
            targets: Optional[SupervisionTargets] = None, background: Optional[torch.Tensor] = None,
            appearance_view: Optional[int] = None, mcmc_num_valid: Optional[int] = None,
            filter_3d: Optional[torch.Tensor] = None) -> None:
        """``targets``: the view's depth and / or mask target ((H, W) float32 CUDA tensors) and, with ``extra_features``, its
        ``labels`` ((H, W) int32) or ``features`` ((H, W, C) float32); ``background``: a (3,) float32 CUDA tensor the image is
        composited on (read on the device when the step runs, so it may be refilled per iteration).  Without supervision
        terms or features this is ``gsb200_train_step``; with supervision terms ``gsb200_train_step_aux``; with features
        ``gsb200_train_step_ext``.  ``appearance_view``: with ``appearance_grids``, the index of the view whose grid slices
        the image and takes an Adam step (``gsb200_train_step_appearance``).  ``mcmc_num_valid``: with ``mcmc``, the number
        of valid rows n_v of the regularisers (``gsb200_train_step_mcmc``); the noise counter is the 0-based iteration.
        ``filter_3d``: the (N,) float32 3D smoothing filter of the rows (``mip_filter.compute_filter_3d``), contiguous, on the
        scene's device; the forward and the backward render through it (``gsb200_train_step_filter3d``)."""
        sc, cfg = self.scene, self.config
        H, W = int(camera_info.camera_height), int(camera_info.camera_width)
        if image_gt.shape != (3, H, W) or not image_gt.is_contiguous() or image_gt.dtype != torch.float32:
            raise ValueError(f"image_gt must be a contiguous float32 (3, {H}, {W}) tensor")
        targets = targets or SupervisionTargets()
        depth_t = targets.depth if self.depth_weight > 0 else None
        mask_t = targets.mask if (self.mask_weight > 0 or background is not None) else None
        if self.depth_weight > 0 and depth_t is None:
            raise ValueError("depth_weight > 0 needs targets.depth")
        if self.mask_weight > 0 and mask_t is None:
            raise ValueError("mask_weight > 0 needs targets.mask")
        for name, x, shape in (("targets.depth", depth_t, (H, W)), ("targets.mask", mask_t, (H, W)),
                               ("background", background, (3,))):
            if x is not None and (tuple(x.shape) != shape or not x.is_contiguous() or x.dtype != torch.float32
                                  or x.device != image_gt.device):
                raise ValueError(f"{name} must be a contiguous float32 {shape} tensor on {image_gt.device}")
        supervised = depth_t is not None or self.mask_weight > 0 or background is not None
        feat_t = None
        if self.extra_features is not None:
            ce = self.feature_loss_kind == "cross_entropy"
            name, feat_t = ("targets.labels", targets.labels) if ce else ("targets.features", targets.features)
            shape, dtype = ((H, W), torch.int32) if ce else ((H, W, self.C), torch.float32)
            if feat_t is None or tuple(feat_t.shape) != shape or not feat_t.is_contiguous() or feat_t.dtype != dtype \
                    or feat_t.device != image_gt.device:
                raise ValueError(f'feature_loss "{self.feature_loss_kind}" needs {name}: a contiguous {dtype} {shape} '
                                 f"tensor on {image_gt.device}")
        if self.appearance_grids is not None:
            V = self.appearance_grids.shape[0]
            if appearance_view is None or not 0 <= int(appearance_view) < V:
                raise ValueError(f"appearance_grids needs appearance_view in 0..{V - 1}, got {appearance_view!r}")
            appearance_view = int(appearance_view)
        elif appearance_view is not None:
            raise ValueError("appearance_view needs appearance_grids")
        if (self.mcmc is None) != (mcmc_num_valid is None):
            raise ValueError("mcmc and mcmc_num_valid must be given together")
        if filter_3d is not None and (tuple(filter_3d.shape) != (self.N,) or filter_3d.dtype != torch.float32
                                      or not filter_3d.is_contiguous() or filter_3d.device != image_gt.device):
            raise ValueError(f"filter_3d must be a contiguous float32 ({self.N},) tensor on {image_gt.device}")
        self._check_previous()
        q, t = q_pointcloud_camera.contiguous(), t_pointcloud_camera.contiguous()
        K = camera_info.camera_intrinsics.contiguous()
        n_obj = q.shape[0]
        b = self._buffers(H, W, n_obj)
        ctl = self.controller
        band = int(color_max_sh_band) if color_max_sh_band in (0, 1, 2) else 3
        self.step_count += 1
        slot = self.step_count % 2
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream(self.device).cuda_stream
            fwd = _lib.GsbForwardArgs(
                num_points=self.N, pointcloud=_ptr(sc.point_cloud), pointcloud_features=_ptr(sc.point_cloud_features),
                point_invalid_mask=_ptr(sc.point_invalid_mask), point_object_id=_ptr(sc.point_object_id), num_objects=n_obj,
                q_pointcloud_camera=_ptr(q), t_pointcloud_camera=_ptr(t), camera_intrinsics=_ptr(K), camera_height=H,
                camera_width=W, near_plane=cfg.near_plane, far_plane=cfg.far_plane,
                depth_to_sort_key_scale=cfg.depth_to_sort_key_scale, rgb_only=0, flags=0, workspace=_ptr(b.ws),
                workspace_bytes=b.layout.total_bytes, key_capacity=self.key_capacity, rasterized_image=_ptr(b.image),
                rasterized_depth=_ptr(b.depth), pixel_accumulated_alpha=_ptr(b.acc_alpha),
                pixel_offset_of_last_effective_point=_ptr(b.last_effective), pixel_valid_point_count=_ptr(b.count), stream=stream,
                host_counters=self._pinned[slot].data_ptr(), host_counters_event=self._events[slot].cuda_event)
            flags = _lib.GSB_FLAG_BACKWARD_TRANSPOSED | (0 if ctl is not None else _lib.GSB_FLAG_NO_HOOK_STATS)
            bwd = _lib.GsbBackwardArgs(
                num_points=self.N, pointcloud=_ptr(sc.point_cloud), pointcloud_features=_ptr(sc.point_cloud_features),
                point_object_id=_ptr(sc.point_object_id), num_objects=n_obj, t_pointcloud_camera=_ptr(t),
                camera_intrinsics=_ptr(K), camera_height=H, camera_width=W, far_plane=cfg.far_plane,
                depth_to_sort_key_scale=cfg.depth_to_sort_key_scale, color_max_sh_band=band, grad_q_factor=cfg.grad_q_factor,
                grad_s_factor=cfg.grad_s_factor, grad_alpha_factor=cfg.grad_alpha_factor, grad_color_factor=cfg.grad_color_factor,
                grad_high_order_color_factor=cfg.grad_high_order_color_factor, flags=flags, workspace=_ptr(b.ws),
                workspace_bytes=b.layout.total_bytes, key_capacity=self.key_capacity, grad_rasterized_image=_ptr(b.grad_image),
                pixel_accumulated_alpha=_ptr(b.acc_alpha), pixel_offset_of_last_effective_point=_ptr(b.last_effective),
                accum=_ptr(self.accum), accum_rows=self.N, grad_pointcloud=_ptr(self.grad_pointcloud),
                grad_pointcloud_features=_ptr(self.grad_pointcloud_features), magnitude_grad_viewspace_on_image=_ptr(b.mag_image),
                stream=stream)
            if ctl is not None:
                bwd.ctl_accumulated_num_in_camera = _ptr(ctl.accumulated_num_in_camera)
                bwd.ctl_accumulated_num_pixels = _ptr(ctl.accumulated_num_pixels)
                bwd.ctl_accumulated_view_space_position_gradients = _ptr(ctl.accumulated_view_space_position_gradients)
                bwd.ctl_accumulated_view_space_position_gradients_avg = _ptr(ctl.accumulated_view_space_position_gradients_avg)
                bwd.ctl_accumulated_position_gradients = _ptr(ctl.accumulated_position_gradients)
                bwd.ctl_accumulated_position_gradients_norm = _ptr(ctl.accumulated_position_gradients_norm)
            args = _lib.GsbTrainStepArgs(
                forward=fwd, backward=bwd, ground_truth_image=_ptr(image_gt), lambda_value=self.lambda_value,
                loss_out3=_ptr(self.loss), loss_temp=_ptr(b.loss_temp), loss_temp_bytes=b.temp_bytes,
                feature_exp_avg=_ptr(self.feature_exp_avg), feature_exp_avg_sq=_ptr(self.feature_exp_avg_sq),
                position_exp_avg=_ptr(self.position_exp_avg), position_exp_avg_sq=_ptr(self.position_exp_avg_sq),
                feature_learning_rate=float(feature_learning_rate), position_learning_rate=float(position_learning_rate),
                beta1=float(self.betas[0]), beta2=float(self.betas[1]), eps=self.eps, step=self.step_count)
            if supervised:
                sup = _lib.GsbSupervisionArgs(
                    depth_target=_ptr(depth_t) if depth_t is not None else None,
                    mask_target=_ptr(mask_t) if mask_t is not None else None,
                    background=_ptr(background) if background is not None else None, depth_weight=self.depth_weight,
                    mask_weight=self.mask_weight, grad_depth=_ptr(b.grad_depth), grad_pixel_accumulated_alpha=_ptr(b.grad_alpha),
                    loss_out3=_ptr(self.supervision_loss), temp=_ptr(b.sup_temp), temp_bytes=b.sup_bytes)
            fx = None
            if feat_t is not None:
                ext = _lib.GsbExtraFeatureArgs(channels=self.C, features=_ptr(self.extra_features), rasterized=_ptr(b.feature_map),
                                               grad_rasterized=_ptr(b.grad_feature_map),
                                               grad_features=_ptr(self.grad_extra_features))
                ce = self.feature_loss_kind == "cross_entropy"
                fx = _lib.GsbFeatureTrainArgs(
                    features=ext, loss_kind=_lib.GSB_FEATURE_LOSS_CROSS_ENTROPY if ce else _lib.GSB_FEATURE_LOSS_L2,
                    weight=self.feature_weight, labels=_ptr(feat_t) if ce else None, target=None if ce else _ptr(feat_t),
                    loss_out2=_ptr(self.feature_loss), temp=_ptr(b.feat_temp), temp_bytes=b.feat_bytes,
                    exp_avg=_ptr(self.extra_feature_exp_avg), exp_avg_sq=_ptr(self.extra_feature_exp_avg_sq),
                    learning_rate=self.extra_feature_learning_rate)
            app = None
            if appearance_view is not None:
                i = appearance_view
                self.appearance_steps[i] += 1
                gz, gy, gx = self.appearance_grids.shape[2:]
                app = _lib.GsbAppearanceArgs(
                    grid=_ptr(self.appearance_grids[i]), grad_grid=_ptr(self.grad_appearance_grid), grid_x=gx, grid_y=gy,
                    grid_z=gz, tv_weight=self.appearance_tv_weight, exp_avg=_ptr(self.appearance_exp_avg[i]),
                    exp_avg_sq=_ptr(self.appearance_exp_avg_sq[i]), learning_rate=self.appearance_learning_rate,
                    step=self.appearance_steps[i], image=_ptr(b.sliced_image), temp=_ptr(b.app_temp), temp_bytes=b.app_bytes,
                    loss_out1=_ptr(self.appearance_tv))
            mcmc_args = None
            if self.mcmc is not None:
                mc = self.mcmc
                mcmc_args = _lib.GsbMcmcStepArgs(
                    num_valid=int(mcmc_num_valid), lambda_opacity=mc.opacity_reg, lambda_scale=mc.scale_reg,
                    noise_scale=mc.noise_lr * float(position_learning_rate), gate_k=GATE_K, min_opacity=mc.min_opacity,
                    seed=int(mc.seed), step=self.step_count - 1, terms_out2=_ptr(self.mcmc_terms), temp=_ptr(self._mcmc_temp))
            if filter_3d is not None:
                _lib.check(self._lib.gsb200_train_step_filter3d(
                    ctypes.byref(args), ctypes.byref(sup) if supervised else None, ctypes.byref(fx) if fx is not None else None,
                    ctypes.byref(app) if app is not None else None,
                    ctypes.byref(mcmc_args) if mcmc_args is not None else None,
                    ctypes.byref(_lib.GsbFilter3dArgs(filter3d=_ptr(filter_3d)))), "gsb200_train_step_filter3d")
            elif mcmc_args is not None:
                _lib.check(self._lib.gsb200_train_step_mcmc(
                    ctypes.byref(args), ctypes.byref(sup) if supervised else None, ctypes.byref(fx) if fx is not None else None,
                    ctypes.byref(app) if app is not None else None, ctypes.byref(mcmc_args)), "gsb200_train_step_mcmc")
            elif app is not None:
                _lib.check(self._lib.gsb200_train_step_appearance(
                    ctypes.byref(args), ctypes.byref(sup) if supervised else None, ctypes.byref(fx) if fx is not None else None,
                    ctypes.byref(app)), "gsb200_train_step_appearance")
            elif fx is not None:
                _lib.check(self._lib.gsb200_train_step_ext(ctypes.byref(args), ctypes.byref(sup) if supervised else None,
                                                           ctypes.byref(fx)), "gsb200_train_step_ext")
            elif supervised:
                _lib.check(self._lib.gsb200_train_step_aux(ctypes.byref(args), ctypes.byref(sup)), "gsb200_train_step_aux")
            else:
                _lib.check(self._lib.gsb200_train_step(ctypes.byref(args)), "gsb200_train_step")
        self._pending[slot] = True
        self._last = SimpleNamespace(buffers=b, H=H, W=W, slot=slot, supervised=supervised,
                                     keep=(q, t, K, image_gt, depth_t, mask_t, background, feat_t, filter_3d))

    @property
    def moments(self) -> MCMCMoments:
        """The Adam moments of this step, for ``GaussianPointMCMCController.refinement``."""
        extra = (self.extra_feature_exp_avg, self.extra_feature_exp_avg_sq) if self.extra_features is not None else None
        return MCMCMoments((self.feature_exp_avg, self.feature_exp_avg_sq), (self.position_exp_avg, self.position_exp_avg_sq),
                           extra)

    # ------------------------------------------------------------------ the latest frame, on demand (these calls wait)
    @property
    def image(self) -> torch.Tensor:
        """(H,W,3) rasterised image of the latest iteration (before the clamp)."""
        return self._last.buffers.image

    @property
    def feature_map(self) -> torch.Tensor:
        """(H,W,C) rendered feature map of the latest iteration (with ``extra_features``)."""
        return self._last.buffers.feature_map

    def hook_input(self) -> "GaussianPointCloudRasterisation.BackwardValidPointHookInput":
        """The latest iteration's ``BackwardValidPointHookInput`` (GPCR:806-817): built only when the controller looks for
        densification candidates (every ``num_iterations_densify`` iterations), never on the per-iteration path."""
        last = self._last
        self._events[last.slot].synchronize()
        pinned = self._pinned[last.slot]
        b = last.buffers
        frame = Frame(b.ws, b.layout, self.N, self.key_capacity, last.H, last.W, 0)
        frame.num_points_in_camera, frame.num_keys = int(pinned[0]), int(pinned[1])
        M = frame.num_points_in_camera
        ids = frame.point_id_in_camera_list
        ids64 = ids.long()
        acc = self.accum[:M]
        return GaussianPointCloudRasterisation.BackwardValidPointHookInput(
            point_id_in_camera_list=ids, grad_point_in_camera=self.grad_pointcloud[ids64],
            grad_pointfeatures_in_camera=self.grad_pointcloud_features[ids64], grad_viewspace=acc[:, 0:2].contiguous(),
            magnitude_grad_viewspace=acc[:, 9].contiguous(), magnitude_grad_viewspace_on_image=b.mag_image,
            num_overlap_tiles=frame.num_overlap_tiles, num_affected_pixels=acc[:, 10].round().to(torch.int32),
            point_uv_in_camera=frame.point_uv.contiguous(), point_depth=frame.point_in_camera[:, 2])
