"""Densification / pruning controller -- consumer of the rasteriser's backward hook (SURVEY §8(f)-1).

Host-side policy code with the reference's names and semantics
(``taichi_3d_gaussian_splatting/GaussianPointAdaptiveController.py:46-393``): fixed-capacity point
cloud with an invalid mask, ``update`` is called from inside the operator's backward with
``BackwardValidPointHookInput`` (GPCR:1127-1142), ``refinement`` after the optimiser step.
The reference implements it with torch tensor ops plus two tiny Taichi kernels
(``compute_ellipsoid_offset`` :10-25, ``sample_from_point`` :27-42); those two are restated with
torch ops here (GaussianPoint3D.py:375-406).  The matplotlib debug plot (:272-288) is not reproduced.
"""
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from .GaussianPointCloudRasterisation import GaussianPointCloudRasterisation
from .utils import quaternion_to_rotation_matrix_torch


def compute_ellipsoid_offset(pointcloud: torch.Tensor, pointcloud_features: torch.Tensor) -> torch.Tensor:
    """Vector from the centre to a focus of each ellipsoid (GaussianPoint3D.py:375-388)."""
    s = pointcloud_features[:, 4:7]
    base = torch.zeros_like(pointcloud)
    sx, sy, sz = s[:, 0], s[:, 1], s[:, 2]
    use_y = (sx < sy) & (sy > sz)
    use_z = (sx < sz) & (sy < sz) & ~use_y
    use_x = ~(use_y | use_z)
    base[use_x, 0] = 1.0
    base[use_y, 1] = 1.0
    base[use_z, 2] = 1.0
    R = quaternion_to_rotation_matrix_torch(pointcloud_features[:, 0:4])
    base = torch.einsum("nij,nj->ni", R, base)
    es = torch.exp(s)
    r_c = es.max(dim=1).values
    r_a = es.min(dim=1).values
    return torch.sqrt(torch.clamp(r_c ** 2 - r_a ** 2, min=0.0))[:, None] * base


def sample_from_point(pointcloud: torch.Tensor, pointcloud_features: torch.Tensor,
                      generator: Optional[torch.Generator] = None) -> torch.Tensor:
    """One sample of N(mean, R S S^T R^T) per point (GaussianPoint3D.py:390-406; the reference draws its
    normals with Box-Muller on ``ti.random``, here with ``torch.randn``)."""
    R = quaternion_to_rotation_matrix_torch(pointcloud_features[:, 0:4])
    es = torch.exp(pointcloud_features[:, 4:7])
    z = torch.randn(pointcloud.shape, device=pointcloud.device, dtype=pointcloud.dtype, generator=generator)
    return pointcloud + torch.einsum("nij,nj->ni", R, es * z)


class GaussianPointAdaptiveController:
    @dataclass
    class GaussianPointAdaptiveControllerConfig:
        # reference: GaussianPointAdaptiveController.py:53-84
        num_iterations_warm_up: int = 500
        num_iterations_densify: int = 100
        transparent_alpha_threshold: float = -0.5
        densification_view_space_position_gradients_threshold: float = 6e-6
        densification_view_avg_space_position_gradients_threshold: float = 1e3
        densification_multi_frame_view_space_position_gradients_threshold: float = 1e3
        densification_multi_frame_view_pixel_avg_space_position_gradients_threshold: float = 1e3
        densification_multi_frame_position_gradients_threshold: float = 1e3
        gaussian_split_factor_phi: float = 1.6
        num_iterations_reset_alpha: int = 3000
        reset_alpha_value: float = 0.1
        floater_num_pixels_threshold: int = 10000
        floater_near_camrea_num_pixels_threshold: int = 10000
        floater_depth_threshold: float = 100
        iteration_start_remove_floater: int = 2000
        plot_densify_interval: int = 200
        under_reconstructed_num_pixels_threshold: int = 512
        under_reconstructed_move_factor: float = 100.0
        enable_ellipsoid_offset: bool = False
        enable_sample_from_point: bool = True

    @dataclass
    class GaussianPointAdaptiveControllerMaintainedParameters:
        pointcloud: torch.Tensor  # [num_points, 3]
        pointcloud_features: torch.Tensor  # [num_points, 56]
        point_invalid_mask: torch.Tensor  # [num_points] int8
        point_object_id: torch.Tensor  # [num_points] int32
        # [num_points, C] or None: per-Gaussian feature vectors (an extension); a clone or split copies its source's row
        point_extra_features: Optional[torch.Tensor] = None

    @dataclass
    class GaussianPointAdaptiveControllerDensifyPointInfo:
        floater_point_id: torch.Tensor
        transparent_point_id: torch.Tensor
        densify_point_id: torch.Tensor
        densify_point_position_before_optimization: torch.Tensor
        densify_size_reduction_factor: torch.Tensor
        densify_point_grad_position: torch.Tensor

    def __init__(self, config: "GaussianPointAdaptiveController.GaussianPointAdaptiveControllerConfig",
                 maintained_parameters: "GaussianPointAdaptiveController.GaussianPointAdaptiveControllerMaintainedParameters",
                 generator: Optional[torch.Generator] = None, verbose: bool = False, fused_update: bool = False):
        """``fused_update``: the per-iteration accumulator update of ``update`` as one CUDA kernel
        (``gsb200_controller_update``) instead of ~15 torch launches (CUDA tensors only)."""
        self.fused_update = fused_update
        self.iteration_counter = -1
        self.config = config
        self.maintained_parameters = maintained_parameters
        self.input_data = None
        self.densify_point_info = None
        self.generator = generator
        self.verbose = verbose
        self.has_plot = False
        self._reset_accumulators()

    def _reset_accumulators(self):
        col = self.maintained_parameters.pointcloud[:, 0]
        self.accumulated_num_pixels = torch.zeros_like(col, dtype=torch.int32)
        self.accumulated_num_in_camera = torch.zeros_like(col, dtype=torch.int32)
        self.accumulated_view_space_position_gradients = torch.zeros_like(col, dtype=torch.float32)
        self.accumulated_view_space_position_gradients_avg = torch.zeros_like(col, dtype=torch.float32)
        self.accumulated_position_gradients = torch.zeros_like(self.maintained_parameters.pointcloud,
                                                               dtype=torch.float32)
        self.accumulated_position_gradients_norm = torch.zeros_like(col, dtype=torch.float32)

    # GaussianPointAdaptiveController.py:130-146
    def update(self, input_data: GaussianPointCloudRasterisation.BackwardValidPointHookInput):
        self.iteration_counter += 1
        if self.fused_update:
            self._update_fused(input_data)
            if self.iteration_counter >= self.config.num_iterations_warm_up and \
                    self.iteration_counter % self.config.num_iterations_densify == 0:
                with torch.no_grad():
                    self._find_densify_points(input_data)
                    self.input_data = input_data
            return
        with torch.no_grad():
            ids = input_data.point_id_in_camera_list.long()
            self.accumulated_num_in_camera[ids] += 1
            self.accumulated_num_pixels[ids] += input_data.num_affected_pixels
            grad_viewspace_norm = input_data.magnitude_grad_viewspace
            self.accumulated_view_space_position_gradients[ids] += grad_viewspace_norm
            avg = grad_viewspace_norm / input_data.num_affected_pixels
            avg[torch.isnan(avg)] = 0
            self.accumulated_view_space_position_gradients_avg[ids] += avg
            self.accumulated_position_gradients[ids] += input_data.grad_point_in_camera
            self.accumulated_position_gradients_norm[ids] += input_data.grad_point_in_camera.norm(dim=1)
            if self.iteration_counter < self.config.num_iterations_warm_up:
                pass
            elif self.iteration_counter % self.config.num_iterations_densify == 0:
                self._find_densify_points(input_data)
                self.input_data = input_data

    def after_fused_update(self, make_hook_input):
        """The accumulators of this iteration were already updated on the device (the fused controller epilogue of the
        per-point backward kernel, ``GsbBackwardArgs.ctl_*``): advance the iteration counter and, on a densification
        iteration only, build the hook tensors (``make_hook_input()``) and pick the candidates like ``update`` does."""
        self.iteration_counter += 1
        if self.iteration_counter >= self.config.num_iterations_warm_up and \
                self.iteration_counter % self.config.num_iterations_densify == 0:
            with torch.no_grad():
                hook = make_hook_input()
                self._find_densify_points(hook)
                self.input_data = hook

    def _update_fused(self, h):
        from . import _lib
        ids = h.point_id_in_camera_list
        if not ids.is_cuda:
            raise RuntimeError("fused_update needs CUDA tensors (there is no CPU path)")
        ids = ids.to(torch.int32).contiguous()
        npix = h.num_affected_pixels.to(torch.int32).contiguous()
        mag = h.magnitude_grad_viewspace.to(torch.float32).contiguous()
        gxyz = h.grad_point_in_camera.to(torch.float32).contiguous()
        with torch.cuda.device(ids.device):
            stream = torch.cuda.current_stream(ids.device).cuda_stream
            _lib.check(_lib.load().gsb200_controller_update(
                ids.data_ptr(), ids.shape[0], npix.data_ptr(), mag.data_ptr(), gxyz.data_ptr(),
                self.accumulated_num_in_camera.data_ptr(), self.accumulated_num_pixels.data_ptr(),
                self.accumulated_view_space_position_gradients.data_ptr(),
                self.accumulated_view_space_position_gradients_avg.data_ptr(),
                self.accumulated_position_gradients.data_ptr(), self.accumulated_position_gradients_norm.data_ptr(),
                stream), "gsb200_controller_update")

    # GaussianPointAdaptiveController.py:148-168
    def refinement(self):
        with torch.no_grad():
            if self.iteration_counter < self.config.num_iterations_warm_up:
                return
            if self.iteration_counter % self.config.num_iterations_densify == 0:
                self._add_densify_points()
                self._reset_accumulators()
            if self.iteration_counter % self.config.num_iterations_reset_alpha == 0:
                self.reset_alpha()
            self.input_data = None

    # ---- selection (reference: GaussianPointAdaptiveController.py:170-270, without the debug plot)
    @staticmethod
    def _safe_div(num: torch.Tensor, den: torch.Tensor) -> torch.Tensor:
        """num / den with 0/0 -> 0 (the reference overwrites NaNs after the division)."""
        out = num / den
        return torch.where(torch.isnan(out), torch.zeros_like(out), out)

    def _removal_masks(self, hook, ids):
        """(floater mask over all points, floater mask over in-camera points, floater ids, transparent mask)."""
        cfg, mp = self.config, self.maintained_parameters
        n = mp.pointcloud.shape[0]
        dev = mp.pointcloud.device
        alive = mp.point_invalid_mask == 0
        floaters_all = torch.zeros(n, dtype=torch.bool, device=dev)
        floaters_cam = torch.zeros(ids.shape[0], dtype=torch.bool, device=dev)
        floater_ids = torch.empty(0, dtype=torch.int64, device=dev)
        if self.iteration_counter > cfg.iteration_start_remove_floater:
            floaters_cam = (hook.num_affected_pixels > cfg.floater_near_camrea_num_pixels_threshold) & \
                (hook.point_depth < cfg.floater_depth_threshold)
            floater_ids = ids[floaters_cam]
            floaters_all[floater_ids] = True
            floaters_all &= alive
        broken = torch.isnan(mp.pointcloud_features).any(dim=1)
        transparent = ((mp.pointcloud_features[:, 7] < cfg.transparent_alpha_threshold) | broken) & alive & ~floaters_all
        return floaters_all, floaters_cam, floater_ids, transparent

    def _find_densify_points(self, hook):
        cfg, mp = self.config, self.maintained_parameters
        n = mp.pointcloud.shape[0]
        dev = mp.pointcloud.device
        ids = hook.point_id_in_camera_list.long()
        floaters_all, floaters_cam, floater_ids, transparent = self._removal_masks(hook, ids)
        doomed = floaters_all | transparent
        doomed_cam = floaters_cam | transparent[ids]

        # this frame: large view-space gradient, or large gradient per covered pixel
        mag = hook.magnitude_grad_viewspace
        pick_cam = (mag > cfg.densification_view_space_position_gradients_threshold) & ~doomed_cam
        pick_cam |= (mag / hook.num_affected_pixels) > cfg.densification_view_avg_space_position_gradients_threshold
        pick_cam &= ~doomed_cam
        picked = torch.zeros(n, dtype=torch.bool, device=dev)
        picked[ids[pick_cam]] = True

        # since the last refinement: the same statistics averaged over the frames a point was seen in
        seen = self.accumulated_num_in_camera
        mean_pixels = self._safe_div(self.accumulated_num_pixels, seen)
        picked |= self._safe_div(self.accumulated_view_space_position_gradients, seen) > \
            cfg.densification_multi_frame_view_space_position_gradients_threshold
        picked |= (self._safe_div(self.accumulated_view_space_position_gradients_avg, seen) / mean_pixels) > \
            cfg.densification_multi_frame_view_pixel_avg_space_position_gradients_threshold
        picked |= (self.accumulated_position_gradients_norm / seen) > \
            cfg.densification_multi_frame_position_gradients_threshold
        picked &= ~doomed
        chosen = torch.nonzero(picked).reshape(-1)

        mean_grad = self._safe_div(self.accumulated_position_gradients[chosen], seen[chosen].unsqueeze(-1))
        shrink = torch.zeros(chosen.shape[0], dtype=torch.float32, device=dev)
        # "over-reconstructed" (covers many pixels) -> split: both halves shrink by phi; otherwise clone
        shrink[self.accumulated_num_pixels[picked] > cfg.under_reconstructed_num_pixels_threshold] = \
            float(np.log(cfg.gaussian_split_factor_phi))
        self.densify_point_info = GaussianPointAdaptiveController.GaussianPointAdaptiveControllerDensifyPointInfo(
            floater_point_id=floater_ids, transparent_point_id=torch.nonzero(transparent).reshape(-1),
            densify_point_id=chosen, densify_point_position_before_optimization=mp.pointcloud[chosen].detach().clone(),
            densify_size_reduction_factor=shrink.unsqueeze(-1), densify_point_grad_position=mean_grad)

    # ---- application (reference: GaussianPointAdaptiveController.py:290-353)
    def _add_densify_points(self):
        assert self.densify_point_info is not None
        cfg, mp, info = self.config, self.maintained_parameters, self.densify_point_info
        xyz, feat, invalid = mp.pointcloud, mp.pointcloud_features, mp.point_invalid_mask
        alive_before = int((invalid == 0).sum())
        invalid[info.transparent_point_id] = 1
        invalid[info.floater_point_id] = 1
        wanted = info.densify_point_id.shape[0]
        slots = torch.nonzero(invalid == 1).reshape(-1)[:wanted]  # freed + spare rows, lowest ids first
        filled = slots.shape[0]
        if filled > 0:
            src = info.densify_point_id[:filled]
            shrink = info.densify_size_reduction_factor[:filled]
            # the copy starts from the source's position BEFORE this optimiser step, so the pair differs
            xyz[slots] = info.densify_point_position_before_optimization[:filled]
            feat[slots] = feat[src]
            mp.point_object_id[slots] = mp.point_object_id[src]
            if mp.point_extra_features is not None:
                mp.point_extra_features[slots] = mp.point_extra_features[src]
            feat[slots, 4:7] -= shrink
            feat[src, 4:7] -= shrink
            split = (shrink > 1e-6).reshape(-1)
            if cfg.enable_ellipsoid_offset:
                shift = compute_ellipsoid_offset(xyz[src], feat[src])
                xyz[slots] += shift
                xyz[src] -= shift
            if cfg.enable_sample_from_point:
                s_src, s_dst = src[split], slots[split]
                xyz[s_dst] = sample_from_point(xyz[s_src], feat[s_src], self.generator)
                xyz[s_src] = sample_from_point(xyz[s_src], feat[s_src], self.generator)
                xyz[slots[~split]] += info.densify_point_grad_position[:filled][~split] * \
                    cfg.under_reconstructed_move_factor
            invalid[slots] = 0
        alive_after = int((invalid == 0).sum())
        assert alive_after == alive_before - info.transparent_point_id.shape[0] - info.floater_point_id.shape[0] + filled
        if self.verbose:
            print(f"valid points {alive_before} -> {alive_after}: {wanted} candidates, {filled} placed, "
                  f"{info.transparent_point_id.shape[0]} transparent, {info.floater_point_id.shape[0]} floaters removed")
        self.densify_point_info = None

    # GaussianPointAdaptiveController.py:355-358
    def reset_alpha(self):
        f = self.maintained_parameters.pointcloud_features
        f[:, 7] = torch.clamp(f[:, 7], max=self.config.reset_alpha_value)
