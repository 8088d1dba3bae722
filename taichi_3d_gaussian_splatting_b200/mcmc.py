"""MCMC densification (Kheradmand et al., "3D Gaussian Splatting as Markov Chain Monte Carlo", NeurIPS 2024): the
alternative to ``densification.GaussianPointAdaptiveController`` with one knob that matters, ``cap_max``.

* every iteration: two L1 regularisers (``loss.mcmc_regulariser``: mean opacity, mean scale of the valid rows) make unused
  Gaussians die, and after the optimiser step a noise shaped by each Gaussian's own covariance is added to its position
  (``add_position_noise``);
* every ``refine_every`` iterations (``refine_start <= t < refine_stop``): dead Gaussians (opacity <= ``min_opacity`` or a
  non-finite feature) are relocated onto live ones drawn with probability proportional to opacity, and the count grows by
  ``grow_factor`` up to ``cap_max`` into invalid rows.  A source drawn k times ends up as n = k + 1 copies whose opacity
  and scale are changed so that the rendered result stays the same (``relocation_opacity_scale``, the paper's eq. 9).

No row is ever invalidated, no tensor is reallocated, there is no opacity reset and no backward-hook statistic is needed.
The exact definition (the Philox counter, the uniform mapping, the Box-Muller pairing) is in ``include/gsb200.h``.  On CUDA
tensors the arithmetic runs in the library's kernels (``csrc/mcmc.cu``); on CPU tensors in the torch forms of this module,
which are also the reference the kernels are tested against.
"""
import ctypes
import math
from dataclasses import dataclass
from typing import Optional, Tuple

import numpy as np
import torch

from .densification import GaussianPointAdaptiveController
from .utils import quaternion_to_rotation_matrix_torch

__all__ = ["MCMCConfig", "MCMCMoments", "GaussianPointMCMCController", "relocation_opacity_scale", "add_position_noise",
           "philox_normals", "N_MAX", "GATE_K"]

N_MAX = 51  # GSB_MCMC_N_MAX of include/gsb200.h
GATE_K = 100.0
_BINOMIAL = torch.tensor([[math.comb(i, k) for k in range(N_MAX)] for i in range(N_MAX)], dtype=torch.float64)


@dataclass
class MCMCConfig:
    cap_max: int  # the budget: the number of valid rows never exceeds min(cap_max, N)
    refine_start: int = 500
    refine_stop: int = 25000
    refine_every: int = 100
    grow_factor: float = 1.05
    min_opacity: float = 0.005
    # the paper's value, for its position learning rate (1.6e-4 decayed to 1.6e-6); not tuned for this trainer's
    # position_learning_rate schedule
    noise_lr: float = 5e5
    opacity_reg: float = 0.01
    scale_reg: float = 0.01
    seed: int = 0  # of the position noise (the draws of a refinement come from the controller's generator)

    def check(self) -> "MCMCConfig":
        if int(self.cap_max) != self.cap_max or self.cap_max < 1:
            raise ValueError(f"cap_max must be a positive integer, got {self.cap_max!r}")
        if not (0 <= self.refine_start <= self.refine_stop) or self.refine_every < 1:
            raise ValueError("the refinement window needs 0 <= refine_start <= refine_stop and refine_every >= 1, got "
                             f"{self.refine_start}, {self.refine_stop}, {self.refine_every}")
        if not (1.0 <= self.grow_factor < float("inf")):
            raise ValueError(f"grow_factor must be finite and >= 1, got {self.grow_factor}")
        if not (0.0 < self.min_opacity < 1.0):
            raise ValueError(f"min_opacity must be in (0, 1), got {self.min_opacity}")
        for name in ("noise_lr", "opacity_reg", "scale_reg"):
            v = getattr(self, name)
            if not (v >= 0.0 and v < float("inf")):
                raise ValueError(f"{name} must be finite and >= 0, got {v}")
        if not 0 <= int(self.seed) < 2 ** 64:
            raise ValueError(f"seed must fit 64 unsigned bits, got {self.seed}")
        return self


def _ptr(t: Optional[torch.Tensor]):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


# ---------------------------------------------------------------------------------------------- position noise
def _philox4x32_10(counter: np.ndarray, key: Tuple[int, int]) -> np.ndarray:
    """Philox4x32-10 of (n, 4) uint32 counters with one 2 x 32-bit key -> (n, 4) uint32."""
    c = [counter[:, k].astype(np.uint64) for k in range(4)]
    k0, k1 = np.uint64(key[0]), np.uint64(key[1])
    mask = np.uint64(0xFFFFFFFF)
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c[0], np.uint64(0xCD9E8D57) * c[2]
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & mask, p1 >> np.uint64(32), p1 & mask
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & mask, (k1 + np.uint64(0xBB67AE85)) & mask
    return np.stack(c, 1).astype(np.uint32)


def philox_normals(num_rows: int, seed: int, step: int) -> np.ndarray:
    """The (num_rows, 3) float64 standard normals eps of ``(seed, step)`` as ``include/gsb200.h`` defines them."""
    i = np.arange(num_rows, dtype=np.uint64)
    counter = np.stack([i & np.uint64(0xFFFFFFFF), i >> np.uint64(32),
                        np.full(num_rows, step & 0xFFFFFFFF, np.uint64), np.full(num_rows, (step >> 32) & 0xFFFFFFFF, np.uint64)],
                       1).astype(np.uint32)
    x = _philox4x32_10(counter, (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF))
    u = ((x >> np.uint32(9)).astype(np.float64) + 0.5) * 2.0 ** -23
    r0, r1 = np.sqrt(-2.0 * np.log(u[:, 0])), np.sqrt(-2.0 * np.log(u[:, 2]))
    return np.stack([r0 * np.cos(2 * np.pi * u[:, 1]), r0 * np.sin(2 * np.pi * u[:, 1]), r1 * np.cos(2 * np.pi * u[:, 3])], 1)


def add_position_noise(point_cloud: torch.Tensor, point_cloud_features: torch.Tensor, point_invalid_mask: torch.Tensor,
                       noise_scale: float, seed: int, step: int, gate_k: float = GATE_K,
                       min_opacity: float = 0.005) -> None:
    """``xyz_i += Sigma_i eps_i noise_scale g(o_i)`` on the valid rows, in place; eps is a pure function of
    ``(seed, step, i)``.  ``noise_scale`` = ``noise_lr`` times the position learning rate of the step."""
    xyz, feat = point_cloud.detach(), point_cloud_features.detach()
    N = xyz.shape[0]
    if xyz.is_cuda:
        from . import _lib
        if xyz.dtype != torch.float32 or not xyz.is_contiguous() or not feat.is_contiguous():
            raise ValueError("the CUDA noise takes contiguous float32 tensors")
        with torch.cuda.device(xyz.device):
            stream = torch.cuda.current_stream(xyz.device).cuda_stream
            _lib.check(_lib.load().gsb200_mcmc_noise(_ptr(xyz), _ptr(feat), _ptr(point_invalid_mask), N, float(noise_scale),
                                                     float(gate_k), float(min_opacity), int(seed), int(step),
                                                     ctypes.c_void_p(stream)), "gsb200_mcmc_noise")
        return
    with torch.no_grad():
        eps = torch.from_numpy(philox_normals(N, int(seed), int(step))).to(xyz.dtype)
        q = feat[:, 0:4]
        R = quaternion_to_rotation_matrix_torch(q / q.norm(dim=1, keepdim=True))
        cov = R @ torch.diag_embed(torch.exp(2 * feat[:, 4:7])) @ R.transpose(1, 2)
        o = torch.sigmoid(feat[:, 7])
        gate = 1 / (1 + torch.exp(-gate_k * ((1 - o) - (1 - min_opacity))))
        delta = torch.einsum("nij,nj->ni", cov, eps) * (noise_scale * gate)[:, None]
        valid = point_invalid_mask == 0
        xyz[valid] += delta[valid]


# ---------------------------------------------------------------------------------------------- relocation arithmetic
def relocation_opacity_scale(logit: torch.Tensor, log_scale: torch.Tensor, n: torch.Tensor,
                             min_opacity: float = 0.005) -> Tuple[torch.Tensor, torch.Tensor]:
    """The logit and log-scales (k, 3) of a Gaussian that becomes ``n`` copies (clamped to ``N_MAX``), evaluated in
    float64: ``o_new = 1 - (1 - o)^(1/n)``, ``s_new = s + log(o / D)``, ``o_new`` clamped to [min_opacity, 1 - 1e-7]."""
    n = n.clamp(1, N_MAX).to(torch.int64)
    o = torch.sigmoid(logit.double())
    o_new = -torch.expm1(torch.log1p(-o) / n.double())
    k = torch.arange(N_MAX, dtype=torch.float64, device=logit.device)
    coef = _BINOMIAL.to(logit.device) * (-1.0) ** k / torch.sqrt(k + 1)  # (i-1, k)
    powers = o_new[:, None] ** (k + 1)  # (m, k)
    inner = powers @ coef.T  # (m, i-1): sum_k C(i-1, k) (-1)^k o_new^(k+1) / sqrt(k+1)
    rows = torch.arange(N_MAX, device=logit.device)[None, :] < n[:, None]
    D = (inner * rows).sum(1)
    oc = o_new.clamp(min_opacity, 1 - 1e-7)
    new_logit = torch.log(oc / (1 - oc)).to(logit.dtype)
    new_log_scale = (log_scale.double() + torch.log(o / D)[:, None]).to(log_scale.dtype)
    return new_logit, new_log_scale


@dataclass
class MCMCMoments:
    """The Adam moments (exp_avg, exp_avg_sq) a refinement has to zero on the rows it touches; any pair may be None."""
    features: Optional[Tuple[torch.Tensor, torch.Tensor]] = None
    positions: Optional[Tuple[torch.Tensor, torch.Tensor]] = None
    extra_features: Optional[Tuple[torch.Tensor, torch.Tensor]] = None

    @staticmethod
    def of_optimizers(feature_optimizer, position_optimizer, extra_optimizer=None) -> "MCMCMoments":
        """The moment tensors of torch-style Adam optimisers over one parameter each (None before their first step)."""
        def pair(opt):
            if opt is None:
                return None
            state = opt.state.get(opt.param_groups[0]["params"][0], {})
            return (state["exp_avg"], state["exp_avg_sq"]) if "exp_avg" in state else None
        return MCMCMoments(pair(feature_optimizer), pair(position_optimizer), pair(extra_optimizer))


class GaussianPointMCMCController:
    MaintainedParameters = GaussianPointAdaptiveController.GaussianPointAdaptiveControllerMaintainedParameters

    def __init__(self, config: MCMCConfig, maintained_parameters, generator: Optional[torch.Generator] = None):
        """``generator``: a ``torch.Generator`` on the scene's device for the draws of the refinements (None: the default
        generator)."""
        self.config = config.check()
        self.maintained_parameters = maintained_parameters
        self.generator = generator
        self.iteration_counter = -1
        self.num_valid = int((maintained_parameters.point_invalid_mask == 0).sum())
        self.last_refinement = None  # (relocated, added) of the latest refinement

    # ------------------------------------------------------------------ once per iteration, after the optimiser step
    def refinement(self, moments: Optional[MCMCMoments] = None) -> None:
        self.iteration_counter += 1
        cfg, t = self.config, self.iteration_counter
        if not (cfg.refine_start <= t < cfg.refine_stop) or t % cfg.refine_every != 0:
            return
        moments = moments or MCMCMoments()
        with torch.no_grad():
            mask = self.maintained_parameters.point_invalid_mask
            dead = torch.nonzero(self._dead()).reshape(-1)
            relocated = self._draw_and_apply(dead, moments) if dead.numel() else 0
            if relocated is None:  # no alive row
                return
            n_v = self.num_valid
            target = min(int(cfg.cap_max), int(math.floor(cfg.grow_factor * n_v)))
            added = 0
            if target > n_v:
                free = torch.nonzero(mask != 0).reshape(-1)[:target - n_v]  # the lowest invalid rows
                if free.numel():
                    added = self._draw_and_apply(free, moments) or 0
            self.num_valid = n_v + added
            self.last_refinement = (relocated, added)

    def _opacity_and_alive(self):
        mp = self.maintained_parameters
        feat = mp.pointcloud_features.detach()
        o = torch.sigmoid(feat[:, 7])
        valid = mp.point_invalid_mask == 0
        alive = valid & (o > self.config.min_opacity) & torch.isfinite(feat).all(dim=1)
        return o, valid, alive

    def _dead(self) -> torch.Tensor:
        _, valid, alive = self._opacity_and_alive()
        return valid & ~alive

    def _draw(self, num: int):
        """``num`` sources from the alive rows with probability proportional to opacity, with replacement:
        (unique source ids, their draw counts, the source of each draw), or None without an alive row."""
        o, _, alive = self._opacity_and_alive()
        alive_ids = torch.nonzero(alive).reshape(-1)
        if alive_ids.numel() == 0:
            return None
        cdf = torch.cumsum(o[alive_ids].double(), 0)
        u = torch.rand(num, dtype=torch.float64, device=cdf.device, generator=self.generator) * cdf[-1]
        idx = torch.searchsorted(cdf, u, right=True).clamp_(max=alive_ids.numel() - 1)
        counts = torch.bincount(idx, minlength=alive_ids.numel())
        drawn = counts > 0
        return alive_ids[drawn], counts[drawn], alive_ids[idx]

    def _draw_and_apply(self, destinations: torch.Tensor, moments: MCMCMoments):
        """Overwrite ``destinations`` with copies of drawn alive rows; the number of rows written, None without an alive row."""
        draw = self._draw(destinations.numel())
        if draw is None:
            return None
        sources, counts, dest_sources = draw
        mp, cfg = self.maintained_parameters, self.config
        xyz, feat = mp.pointcloud.detach(), mp.pointcloud_features.detach()
        extra = mp.point_extra_features.detach() if mp.point_extra_features is not None else None
        if xyz.is_cuda:
            self._apply_cuda(sources, counts, destinations, dest_sources, xyz, feat, extra, moments)
        else:
            logit, log_scale = relocation_opacity_scale(feat[sources, 7], feat[sources, 4:7], counts + 1, cfg.min_opacity)
            feat[sources, 7] = logit
            feat[sources, 4:7] = log_scale
            xyz[destinations] = xyz[dest_sources]
            feat[destinations] = feat[dest_sources]
            mp.point_object_id[destinations] = mp.point_object_id[dest_sources]
            if extra is not None:
                extra[destinations] = extra[dest_sources]
            mp.point_invalid_mask[destinations] = 0
            for pair in (moments.features, moments.positions, moments.extra_features):
                for m in pair or ():
                    m[sources] = 0
                    m[destinations] = 0
        return int(destinations.numel())

    def _apply_cuda(self, sources, counts, destinations, dest_sources, xyz, feat, extra, moments: MCMCMoments):
        from . import _lib
        mp = self.maintained_parameters
        i32 = lambda x: x.to(torch.int32).contiguous()  # noqa: E731
        sources, counts, destinations, dest_sources = i32(sources), i32(counts), i32(destinations), i32(dest_sources)
        fm, pm, em = (pair or (None, None) for pair in (moments.features, moments.positions, moments.extra_features))
        with torch.cuda.device(xyz.device):
            args = _lib.GsbMcmcRelocateArgs(
                num_points=xyz.shape[0], num_sources=sources.numel(), source_ids=_ptr(sources), source_counts=_ptr(counts),
                num_destinations=destinations.numel(), destination_ids=_ptr(destinations),
                destination_sources=_ptr(dest_sources), pointcloud=_ptr(xyz), pointcloud_features=_ptr(feat),
                point_invalid_mask=_ptr(mp.point_invalid_mask), point_object_id=_ptr(mp.point_object_id),
                extra_features=_ptr(extra), channels=extra.shape[1] if extra is not None else 0,
                min_opacity=self.config.min_opacity, feature_exp_avg=_ptr(fm[0]), feature_exp_avg_sq=_ptr(fm[1]),
                position_exp_avg=_ptr(pm[0]), position_exp_avg_sq=_ptr(pm[1]), extra_exp_avg=_ptr(em[0]),
                extra_exp_avg_sq=_ptr(em[1]), stream=torch.cuda.current_stream(xyz.device).cuda_stream)
            _lib.check(_lib.load().gsb200_mcmc_relocate(ctypes.byref(args)), "gsb200_mcmc_relocate")
