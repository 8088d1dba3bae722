"""Training loss of the reference trainer (SURVEY §8(f)-3): ``L = (1 - lambda) * L1 + lambda * (1 - SSIM)``
(+ optional exp(s) regulariser), same class / config names as
``taichi_3d_gaussian_splatting/LossFunction.py:8-54``.

The reference takes SSIM from the third-party ``pytorch_msssim`` package (``requirements.txt:4``, unpinned,
not installed in this image); its published algorithm is restated here: 11x11 Gaussian window with
sigma = 1.5 applied separably with VALID padding, K1 = 0.01, K2 = 0.03, ``data_range = 1``,
``size_average = True`` (mean over channels and batch), no non-negative clamp.  No reference test touches
the loss, so its parity is unpinned (SURVEY §8(f)-3).
"""
from dataclasses import dataclass
from typing import Callable, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F


def _gaussian_window(size: int, sigma: float, device, dtype) -> torch.Tensor:
    coords = torch.arange(size, device=device, dtype=dtype) - size // 2
    g = torch.exp(-(coords ** 2) / (2 * sigma ** 2))
    return g / g.sum()


def _filter(x: torch.Tensor, win: torch.Tensor) -> torch.Tensor:
    c = x.shape[1]
    k = win.numel()
    out = F.conv2d(x, win.view(1, 1, k, 1).expand(c, 1, k, 1), groups=c)
    return F.conv2d(out, win.view(1, 1, 1, k).expand(c, 1, 1, k), groups=c)


def ssim(x: torch.Tensor, y: torch.Tensor, data_range: float = 1.0, size_average: bool = True,
         win_size: int = 11, win_sigma: float = 1.5, K=(0.01, 0.03)) -> torch.Tensor:
    """Structural similarity of (B, C, H, W) images (H, W > win_size - 1)."""
    win = _gaussian_window(win_size, win_sigma, x.device, x.dtype)
    c1, c2 = (K[0] * data_range) ** 2, (K[1] * data_range) ** 2
    mu1, mu2 = _filter(x, win), _filter(y, win)
    mu1_sq, mu2_sq, mu12 = mu1 * mu1, mu2 * mu2, mu1 * mu2
    s1 = _filter(x * x, win) - mu1_sq
    s2 = _filter(y * y, win) - mu2_sq
    s12 = _filter(x * y, win) - mu12
    cs_map = (2 * s12 + c2) / (s1 + s2 + c2)
    ssim_map = ((2 * mu12 + c1) / (mu1_sq + mu2_sq + c1)) * cs_map
    per_channel = ssim_map.flatten(2).mean(-1)
    return per_channel.mean() if size_average else per_channel.mean(1)


_l1_temp = {}


def fused_l1_loss_with_grad(predicted_image: torch.Tensor, ground_truth_image: torch.Tensor, clamp01: bool = False,
                            weight: float = 1.0, want_grad: bool = True):
    """``weight * mean|clamp01(pred) - gt|`` and its gradient w.r.t. ``pred`` in ONE CUDA kernel
    (``gsb200_l1_loss``; clamp of GaussianPointTrainer.py:168-170 + L1 of LossFunction.py:29).
    Returns ``(loss, grad)``: ``loss`` is a 0-dim device tensor holding the UNWEIGHTED mean, ``grad`` already
    carries ``weight`` -- feed it to ``image.backward(grad)``.  CUDA float32 contiguous tensors only: there is
    no CPU path."""
    from . import _lib
    if not (predicted_image.is_cuda and ground_truth_image.is_cuda):
        raise RuntimeError("fused_l1_loss_with_grad needs CUDA tensors (there is no CPU path)")
    if predicted_image.dtype != torch.float32 or ground_truth_image.dtype != torch.float32:
        raise RuntimeError("fused_l1_loss_with_grad needs float32 tensors")
    if predicted_image.shape != ground_truth_image.shape:
        raise RuntimeError("fused_l1_loss_with_grad: shape mismatch")
    pred = predicted_image.detach().contiguous()
    gt = ground_truth_image.detach().contiguous()
    lib = _lib.load()
    stream = torch.cuda.current_stream(pred.device)
    key = (pred.device.index, stream.cuda_stream)
    temp = _l1_temp.get(key)
    if temp is None:
        temp = torch.zeros(int(lib.gsb200_l1_loss_temp_bytes()), dtype=torch.uint8, device=pred.device)
        _l1_temp[key] = temp
    loss = torch.empty((), dtype=torch.float32, device=pred.device)
    grad = torch.empty_like(pred) if want_grad else None
    _lib.check(lib.gsb200_l1_loss(pred.data_ptr(), gt.data_ptr(), pred.numel(), int(bool(clamp01)), float(weight),
                                  loss.data_ptr(), grad.data_ptr() if want_grad else None, temp.data_ptr(),
                                  temp.numel(), stream.cuda_stream), "gsb200_l1_loss")
    return loss, grad


class _FusedL1(torch.autograd.Function):
    @staticmethod
    def forward(ctx, predicted_image, ground_truth_image, clamp01):
        loss, grad = fused_l1_loss_with_grad(predicted_image, ground_truth_image, clamp01,
                                             want_grad=predicted_image.requires_grad)
        ctx.grad = grad
        return loss

    @staticmethod
    def backward(ctx, grad_output):
        grad = ctx.grad
        ctx.grad = None
        return (grad * grad_output if grad is not None else None), None, None


def fused_l1_loss(predicted_image: torch.Tensor, ground_truth_image: torch.Tensor, clamp01: bool = False):
    """Differentiable form of :func:`fused_l1_loss_with_grad` (one extra scaling kernel in backward)."""
    return _FusedL1.apply(predicted_image, ground_truth_image, clamp01)


_image_loss_temp = {}


def fused_image_loss_with_grad(rasterized_image: torch.Tensor, ground_truth_image: torch.Tensor, lambda_value: float = 0.2,
                               weight: float = 1.0, want_grad: bool = True):
    """The trainer's whole image loss in two CUDA kernels (``gsb200_image_loss``, csrc/image_loss.cu):
    ``pred = clamp(rasterized_image, 0, 1)`` (GaussianPointTrainer.py:168-170), ``L = (1 - lambda) * L1 + lambda *
    (1 - SSIM)`` (LossFunction.py:29-33) and ``weight * dL/d rasterized_image``.  ``rasterized_image`` is the (H, W, 3)
    tensor the rasteriser returns (no permute), ``ground_truth_image`` the (3, H, W) tensor of the dataset.  Returns
    ``(losses, grad)``: ``losses`` a device tensor ``[L, L1, 1 - SSIM]`` (unweighted), ``grad`` (H, W, 3) or None --
    feed it to ``rasterized_image.backward(grad)``.  CUDA float32 tensors only: there is no CPU path."""
    from . import _lib
    if not (rasterized_image.is_cuda and ground_truth_image.is_cuda):
        raise RuntimeError("fused_image_loss_with_grad needs CUDA tensors (there is no CPU path)")
    if rasterized_image.dtype != torch.float32 or ground_truth_image.dtype != torch.float32:
        raise RuntimeError("fused_image_loss_with_grad needs float32 tensors")
    if rasterized_image.dim() != 3 or rasterized_image.shape[2] != 3:
        raise RuntimeError("rasterized_image must be (H, W, 3)")
    H, W = int(rasterized_image.shape[0]), int(rasterized_image.shape[1])
    if tuple(ground_truth_image.shape) != (3, H, W):
        raise RuntimeError(f"ground_truth_image must be (3, {H}, {W}), got {tuple(ground_truth_image.shape)}")
    if H <= 10 or W <= 10:
        raise RuntimeError("images must be larger than the 11-tap SSIM window")
    pred = rasterized_image.detach().contiguous()
    gt = ground_truth_image.detach().contiguous()
    lib = _lib.load()
    stream = torch.cuda.current_stream(pred.device)
    key = (pred.device.index, stream.cuda_stream, H, W)
    temp = _image_loss_temp.get(key)
    if temp is None:
        temp = torch.zeros(int(lib.gsb200_image_loss_temp_bytes(H, W)), dtype=torch.uint8, device=pred.device)
        _image_loss_temp[key] = temp
    losses = torch.empty((3,), dtype=torch.float32, device=pred.device)
    grad = torch.empty_like(pred) if want_grad else None
    _lib.check(lib.gsb200_image_loss(pred.data_ptr(), gt.data_ptr(), H, W, float(lambda_value), float(weight),
                                     losses.data_ptr(), grad.data_ptr() if want_grad else None, temp.data_ptr(),
                                     temp.numel(), stream.cuda_stream), "gsb200_image_loss")
    return losses, grad


class _FusedImageLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, rasterized_image, ground_truth_image, lambda_value):
        losses, grad = fused_image_loss_with_grad(rasterized_image, ground_truth_image, lambda_value,
                                                  want_grad=rasterized_image.requires_grad)
        ctx.grad = grad
        loss, l1, ld_ssim = losses[0], losses[1], losses[2]
        ctx.mark_non_differentiable(l1, ld_ssim)
        return loss, l1, ld_ssim

    @staticmethod
    def backward(ctx, grad_loss, grad_l1, grad_dssim):
        grad = ctx.grad
        ctx.grad = None
        return (grad * grad_loss if grad is not None else None), None, None


def fused_image_loss(rasterized_image: torch.Tensor, ground_truth_image: torch.Tensor, lambda_value: float = 0.2):
    """Differentiable form of :func:`fused_image_loss_with_grad`: ``(L, L1, 1 - SSIM)`` as 0-dim tensors, ``L`` carrying
    the gradient to ``rasterized_image`` (one extra scaling kernel in backward)."""
    return _FusedImageLoss.apply(rasterized_image, ground_truth_image, lambda_value)


@dataclass
class SupervisionTargets:
    """Optional per-view targets besides the image: ``depth`` (H, W) float32 in point-cloud units along the optical axis
    (0 or NaN = no measurement, e.g. sparse LiDAR) and ``mask`` (H, W) float32 in [0, 1] (1 = object); for a loss on the
    rendered per-Gaussian feature map (:func:`feature_loss`), ``labels`` (H, W) int32 class ids (outside [0, C) = no label)
    or ``features`` (H, W, C) float32 (a pixel with a non-finite value = no target); ``loss_weight`` (H, W) float32 in [0, 1],
    a static per-pixel weight of the image loss (0 = ignore the pixel; :func:`robust_weight`)."""
    depth: Optional[torch.Tensor] = None
    mask: Optional[torch.Tensor] = None
    labels: Optional[torch.Tensor] = None
    features: Optional[torch.Tensor] = None
    loss_weight: Optional[torch.Tensor] = None


FEATURE_LOSSES = ("cross_entropy", "l2")


def feature_loss(feature_map: torch.Tensor, targets: SupervisionTargets, kind: str, weight: float) -> torch.Tensor:
    """The loss on the rendered (H, W, C) feature map ``F`` (the operator's ``point_extra_features`` output); the fused train
    step (``gsb200_train_step_ext`` / ``csrc/feature_loss.cu``) computes the same:

    * ``"cross_entropy"`` (semantic labels, C >= 2): ``weight * sum_labelled CE(softmax(F_p), label_p) / max(n_labelled, 1)``
      on ``targets.labels`` (H, W) int32, a pixel labelled when ``0 <= label < C``;
    * ``"l2"`` (distilled feature maps): ``weight * sum_supervised sum_c (F_pc - T_pc)^2 / max(n_supervised * C, 1)`` on
      ``targets.features`` (H, W, C), a pixel supervised when all C of its values are finite.

    Unsupervised pixels contribute nothing and get a zero gradient.  Returns the term as a 0-dim tensor."""
    C = feature_map.shape[-1]
    if kind == "cross_entropy":
        if targets.labels is None:
            raise ValueError('feature loss "cross_entropy" needs targets.labels')
        if C < 2:
            raise ValueError(f'feature loss "cross_entropy" needs C >= 2 channels, got {C}')
        labels = targets.labels.long()
        valid = (labels >= 0) & (labels < C)
        safe = torch.where(valid, labels, torch.zeros_like(labels))
        nll = -torch.log_softmax(feature_map, dim=-1).gather(-1, safe[..., None])[..., 0]  # max-subtracted log-sum-exp
        err = torch.where(valid, nll, torch.zeros_like(nll))
        return weight * err.sum() / valid.sum().clamp_min(1)
    if kind == "l2":
        if targets.features is None:
            raise ValueError('feature loss "l2" needs targets.features')
        T = targets.features
        valid = torch.isfinite(T).all(dim=-1)
        safe = torch.where(valid[..., None], T, torch.zeros_like(T))  # no NaN reaches the gradient of the unused branch
        err = torch.where(valid[..., None], (feature_map - safe) ** 2, torch.zeros_like(T))
        return weight * err.sum() / (valid.sum() * C).clamp_min(1)
    raise ValueError(f"feature loss must be one of {FEATURE_LOSSES}, got {kind!r}")


def _torch_image_loss(rasterized_image, ground_truth_image, lambda_value):
    """clamp + (1 - lambda) L1 + lambda (1 - SSIM) of the (H, W, 3) image against the (3, H, W) ground truth."""
    pred = torch.clamp(rasterized_image, min=0, max=1).permute(2, 0, 1)[None]
    gt = ground_truth_image[None]
    l1 = torch.abs(pred - gt).mean()
    ld_ssim = 1 - ssim(pred, gt, data_range=1, size_average=True)
    return (1 - lambda_value) * l1 + lambda_value * ld_ssim, l1, ld_ssim


ROBUST_BINS = 4096
ROBUST_PATCH = 16


@dataclass
class RobustLossConfig:
    """The trimmed robust image loss of RobustNeRF (Sabour et al., "RobustNeRF: Ignoring Distractors with Robust Losses",
    CVPR 2023, section 4), which drops the pixels of transient distractors (people, cars, shadows that are in one view and
    not the next) from the image loss: :func:`robust_weight` states it.  ``inlier_quantile`` q in (0, 1]: the residual
    quantile below which a pixel is a raw inlier; ``box_threshold`` and ``patch_threshold`` in [0, 1]: the fraction of raw
    inliers a pixel's 3x3 neighbourhood, and of 3x3 inliers a 16x16 patch, needs for the pixel to count as an inlier;
    ``start_iteration``: the first training iteration that applies the mask (before it, only static weights do).

    RobustNeRF's values as we read section 4 are the median residual (q = 0.5), a 3x3 box threshold of 0.5 and a 16x16 patch
    threshold of 0.6, with a pixel kept when its 3x3 rule or its patch rule keeps it; the thresholds and the rule are the
    defaults here.  The default quantile is 0.9, a choice of this project: on the distractor fit of
    ``tests/test_gpu_robust_loss.py`` (12 views at 128x192 with two opaque boxes each, 600 fused iterations, mask from
    iteration 100; NVIDIA H100 80GB HBM3, 700 W power limit) PSNR against clean renders of the training / held-out poses was
    41.80 / 42.00 dB without the mask, 33.66 / 33.94 dB with q = 0.5, 37.30 / 37.82 dB with q = 0.7 and 42.54 / 42.84 dB with
    q = 0.9 (static weights over the boxes: 42.80 / 42.92 dB): trimming half of every view also drops much of the scene once
    the fit is good.  Other choices of this project: the quantile is taken over one whole view's pixels rather than over a batch of rays drawn from many views; the
    patches are the image's fixed 16x16 tiles (the rasteriser's tiles), not patches sampled at random; pixels with static
    weight 0 are left out of every count; and the residual is the mean absolute error over the three channels of the clamped
    image (the paper uses the squared error of its L2 loss; the order of the residuals, all that the quantile sees, is the
    same for one channel)."""
    inlier_quantile: float = 0.9
    box_threshold: float = 0.5
    patch_threshold: float = 0.6
    start_iteration: int = 0

    def __post_init__(self):
        q = self.inlier_quantile
        if not (isinstance(q, (int, float)) and 0.0 < q <= 1.0):
            raise ValueError(f"inlier_quantile must be in (0, 1], got {q!r}")
        for name in ("box_threshold", "patch_threshold"):
            v = getattr(self, name)
            if not (isinstance(v, (int, float)) and 0.0 <= v <= 1.0):
                raise ValueError(f"{name} must be in [0, 1], got {v!r}")
        if not (isinstance(self.start_iteration, int) and self.start_iteration >= 0):
            raise ValueError(f"start_iteration must be an int >= 0, got {self.start_iteration!r}")


def robust_weight(image: torch.Tensor, ground_truth_image: torch.Tensor, static_weight: Optional[torch.Tensor] = None,
                  config: Optional[RobustLossConfig] = None):
    """The per-pixel weight ``w`` (H, W) of the image loss, for the (H, W, 3) image ``x`` the image loss reads (after the
    background composite and the appearance grid) and its (3, H, W) ground truth ``g``; H and W multiples of 16.  With
    ``s`` the static weight (1 everywhere when None):

    * residual ``r = (|c0 - g0| + |c1 - g1| + |c2 - g2|) / 3`` in float32 in this order, ``c = clamp(x, 0, 1)``;
    * ``bin = min(floor(4096 r), 4095)``; ``b`` = the smallest bin with ``(float)cum(b) >= q (float)n``, ``cum`` the
      histogram of the bins of the ``n`` pixels with ``s > 0``; a pixel is a raw inlier when ``bin <= b``;
    * 3x3 inlier: ``(float)#raw inliers >= box_threshold (float)#neighbours`` over its in-image 3x3 neighbours with s > 0;
    * patch inlier: every pixel of a 16x16 tile when ``(float)#3x3 inliers >= patch_threshold (float)#pixels`` over the
      tile's pixels with s > 0;
    * ``w = s [3x3 inlier or patch inlier]``; without ``config``, ``w = s``.

    Returns ``(w, stats)``: ``stats`` a (2,) float32 tensor {inlier fraction ``sum[w > 0 among s > 0] / n`` (0 when n = 0),
    threshold ``(b + 1) / 4096``, 1 without ``config``}.  Exact integer work and float32 comparisons: the CUDA kernels
    (``csrc/robust_loss.cu``) reproduce it bit for bit.  Not differentiated."""
    with torch.no_grad():
        H, W = int(image.shape[0]), int(image.shape[1])
        if H % ROBUST_PATCH or W % ROBUST_PATCH or H == 0 or W == 0:
            raise ValueError(f"the loss weights need H and W to be multiples of {ROBUST_PATCH}, got {H}x{W}")
        f32 = lambda v: torch.tensor(v, dtype=torch.float32, device=image.device)  # noqa: E731
        s = torch.ones((H, W), dtype=torch.float32, device=image.device) if static_weight is None else static_weight
        valid = s > 0
        n = int(valid.sum())
        if config is None:
            w = s.clone()
            threshold = 1.0
        else:
            c = torch.clamp(image, 0, 1)
            d = torch.abs(c - ground_truth_image.permute(1, 2, 0))
            r = (d[..., 0] + d[..., 1] + d[..., 2]) / f32(3.0)  # a tensor divisor: a true division on every device
            bins = torch.clamp(torch.floor(r * ROBUST_BINS), max=ROBUST_BINS - 1).long()
            cum = torch.bincount(bins[valid], minlength=ROBUST_BINS).cumsum(0)
            b = int(torch.nonzero(cum.to(torch.float32) >= f32(config.inlier_quantile) * f32(float(n)))[0, 0])
            raw = valid & (bins <= b)
            pad = lambda m: F.pad(m.to(torch.int32)[None, None], (1, 1, 1, 1))[0, 0]  # noqa: E731
            pv, pr = pad(valid), pad(raw)
            cnt = sum(pv[i:i + H, j:j + W] for i in range(3) for j in range(3))
            inl = sum(pr[i:i + H, j:j + W] for i in range(3) for j in range(3))
            box = inl.to(torch.float32) >= f32(config.box_threshold) * cnt.to(torch.float32)
            tiles = lambda m: m.to(torch.int32).reshape(H // 16, 16, W // 16, 16).sum(dim=(1, 3))  # noqa: E731
            patch = tiles(valid & box).to(torch.float32) >= f32(config.patch_threshold) * tiles(valid).to(torch.float32)
            patch = patch.repeat_interleave(16, 0).repeat_interleave(16, 1)
            w = s * (box | patch).to(torch.float32)
            threshold = (b + 1) / ROBUST_BINS
        kept = int((valid & (w > 0)).sum())
        stats = torch.tensor([kept / n if n else 0.0, threshold], dtype=torch.float32, device=image.device)
    return w, stats


def robust_composite(image: torch.Tensor, ground_truth_image: torch.Tensor, weight: torch.Tensor) -> torch.Tensor:
    """``x' = w c + (1 - w) g`` (H, W, 3), ``c = clamp(image, 0, 1)``: the image the image loss reads under the per-pixel
    weight ``w`` (H, W).  A pixel of weight 0 is its ground truth, so it adds nothing to the L1 or the D-SSIM term and no
    SSIM window hands it a gradient; the gradient to ``image`` is ``w 1[0 <= x <= 1] dL/dx'``.  The normalisation stays
    over all pixels."""
    w = weight[..., None]
    return w * torch.clamp(image, 0, 1) + (1 - w) * ground_truth_image.permute(1, 2, 0)


_robust_temp = {}


def fused_robust_image_loss_with_grad(rasterized_image: torch.Tensor, ground_truth_image: torch.Tensor,
                                      lambda_value: float = 0.2, static_weight: Optional[torch.Tensor] = None,
                                      config: Optional[RobustLossConfig] = None):
    """:func:`fused_image_loss_with_grad` under the per-pixel weights of :func:`robust_weight` in CUDA kernels
    (``gsb200_robust_image_loss``, csrc/robust_loss.cu around the unchanged image-loss kernels).  Returns ``(losses, grad,
    weight, stats)``: the image loss ``[L, L1, 1 - SSIM]`` of the composite, dL/d rasterized_image (H, W, 3), ``w`` (H, W)
    and {inlier fraction, threshold}.  CUDA float32 tensors only: there is no CPU path."""
    from . import _lib
    if not (rasterized_image.is_cuda and ground_truth_image.is_cuda):
        raise RuntimeError("fused_robust_image_loss_with_grad needs CUDA tensors (there is no CPU path)")
    if rasterized_image.dim() != 3 or rasterized_image.shape[2] != 3 or rasterized_image.dtype != torch.float32:
        raise RuntimeError("rasterized_image must be a float32 (H, W, 3) tensor")
    H, W = int(rasterized_image.shape[0]), int(rasterized_image.shape[1])
    if tuple(ground_truth_image.shape) != (3, H, W) or ground_truth_image.dtype != torch.float32:
        raise RuntimeError(f"ground_truth_image must be a float32 (3, {H}, {W}) tensor")
    if ground_truth_image.device != rasterized_image.device:
        raise RuntimeError(f"ground_truth_image must be on {rasterized_image.device}")
    if static_weight is not None and (tuple(static_weight.shape) != (H, W) or static_weight.dtype != torch.float32
                                      or static_weight.device != rasterized_image.device):
        raise RuntimeError(f"static_weight must be a float32 ({H}, {W}) tensor on {rasterized_image.device}")
    pred = rasterized_image.detach().contiguous()
    gt = ground_truth_image.detach().contiguous()
    sw = None if static_weight is None else static_weight.detach().contiguous()
    lib = _lib.load()
    stream = torch.cuda.current_stream(pred.device)
    key = (pred.device.index, stream.cuda_stream, H, W)
    temps = _robust_temp.get(key)
    if temps is None:
        il_bytes, rl_bytes = int(lib.gsb200_image_loss_temp_bytes(H, W)), int(lib.gsb200_robust_temp_bytes(H, W))
        temps = (torch.zeros(il_bytes, dtype=torch.uint8, device=pred.device),
                 torch.zeros(max(rl_bytes, 16), dtype=torch.uint8, device=pred.device))
        _robust_temp[key] = temps
    losses = torch.empty((3,), dtype=torch.float32, device=pred.device)
    grad = torch.empty_like(pred)
    weight = torch.empty((H, W), dtype=torch.float32, device=pred.device)
    composite = torch.empty_like(pred)
    stats = torch.empty((2,), dtype=torch.float32, device=pred.device)
    cfg = config or RobustLossConfig()
    args = _lib.GsbRobustLossArgs(static_weight=None if sw is None else sw.data_ptr(), robust=int(config is not None),
                                  inlier_quantile=cfg.inlier_quantile, box_threshold=cfg.box_threshold,
                                  patch_threshold=cfg.patch_threshold, weight_out=weight.data_ptr(),
                                  composite=composite.data_ptr(), temp=temps[1].data_ptr(), temp_bytes=temps[1].numel(),
                                  stats_out2=stats.data_ptr())
    import ctypes
    _lib.check(lib.gsb200_robust_image_loss(pred.data_ptr(), gt.data_ptr(), H, W, float(lambda_value), ctypes.byref(args),
                                            losses.data_ptr(), grad.data_ptr(), temps[0].data_ptr(), temps[0].numel(),
                                            stream.cuda_stream), "gsb200_robust_image_loss")
    return losses, grad, weight, stats


def supervision_loss(image: torch.Tensor, depth: Optional[torch.Tensor], alpha: Optional[torch.Tensor],
                     ground_truth_image: torch.Tensor, targets: Optional[SupervisionTargets] = None,
                     background: Optional[torch.Tensor] = None, lambda_value: float = 0.2, depth_weight: float = 0.0,
                     mask_weight: float = 0.0, image_loss: Optional[Callable] = None):
    """The training loss with the optional depth, mask and background terms, for one view (the fused train step,
    ``gsb200_train_step_aux`` / ``csrc/supervision_loss.cu``, computes the same):

    * background ``bg`` (3,) given: the image loss runs on ``I' = image + (1 - alpha)[..., None] * bg``; with a mask the
      ground truth is composited as well, ``gt' = gt * m + (1 - m) * bg``; without one it is taken to be on ``bg``;
    * mask term ``mask_weight * mean |alpha - m|``;
    * depth term ``depth_weight * sum_valid |depth - d*| / max(n_valid, 1)``, valid where ``d*`` is finite and > 0.

    ``image`` (H, W, 3) unclamped as the rasteriser returns it, ``depth`` / ``alpha`` (H, W) (only needed by the terms that
    use them), ``ground_truth_image`` (3, H, W).  ``image_loss(I', gt') -> (L, L1, 1 - SSIM)`` defaults to clamp +
    ``(1 - lambda) L1 + lambda (1 - SSIM)`` in torch.  Returns ``(total, L1, 1 - SSIM, mask term, depth term)``; a term
    that is off is a zero tensor."""
    targets = targets or SupervisionTargets()
    mask = targets.mask
    gt = ground_truth_image
    if background is not None:
        bg = background.to(image.dtype)
        image = image + (1 - alpha)[..., None] * bg
        if mask is not None:
            gt = gt * mask[None] + (1 - mask)[None] * bg[:, None, None]
    if image_loss is None:
        loss, l1, ld_ssim = _torch_image_loss(image, gt, lambda_value)
    else:
        loss, l1, ld_ssim = image_loss(image, gt)
    zero = torch.zeros((), dtype=image.dtype, device=image.device)
    mask_term = depth_term = zero
    if mask_weight > 0:
        if mask is None:
            raise ValueError("mask_weight > 0 needs a mask target")
        mask_term = mask_weight * torch.abs(alpha - mask).mean()
    if depth_weight > 0:
        if targets.depth is None:
            raise ValueError("depth_weight > 0 needs a depth target")
        d = targets.depth
        valid = torch.isfinite(d) & (d > 0)
        safe = torch.where(valid, d, torch.zeros_like(d))  # no NaN reaches the gradient of the unused branch
        err = torch.where(valid, torch.abs(depth - safe), torch.zeros_like(d))
        depth_term = depth_weight * err.sum() / valid.sum().clamp_min(1)
    return loss + mask_term + depth_term, l1, ld_ssim, mask_term, depth_term


class LossFunction(nn.Module):
    @dataclass
    class LossFunctionConfig:
        lambda_value: float = 0.2
        enable_regularization: bool = True
        regularization_weight: float = 2

    def __init__(self, config: "LossFunction.LossFunctionConfig"):
        super().__init__()
        self.config = config

    def forward_rasterized(self, rasterized_image, ground_truth_image, point_invalid_mask=None, pointcloud_features=None):
        """The trainer-step form of ``forward`` on the rasteriser's own (H, W, 3) output, UNclamped, against the dataset's
        (3, H, W) image: clamp (GaussianPointTrainer.py:168-170) + loss in two fused CUDA kernels instead of ~60 autograd
        kernels.  Same return value as ``forward(clamp(rasterized_image).permute(2, 0, 1), ground_truth_image, ...)``."""
        loss, l1, ld_ssim = fused_image_loss(rasterized_image, ground_truth_image, self.config.lambda_value)
        if pointcloud_features is not None and self.config.enable_regularization:
            s = pointcloud_features[point_invalid_mask == 0, 4:7]
            loss = loss + self.config.regularization_weight * torch.norm(torch.exp(s), dim=1).mean()
        return loss, l1, ld_ssim

    def forward(self, predicted_image, ground_truth_image, point_invalid_mask=None, pointcloud_features=None):
        """predicted / ground truth: (B, C, H, W) or (C, H, W).  Returns (L, L1, 1 - SSIM)."""
        if predicted_image.dim() == 3:
            predicted_image = predicted_image.unsqueeze(0)
        if ground_truth_image.dim() == 3:
            ground_truth_image = ground_truth_image.unsqueeze(0)
        l1 = torch.abs(predicted_image - ground_truth_image).mean()
        ld_ssim = 1 - ssim(predicted_image, ground_truth_image, data_range=1, size_average=True)
        loss = (1 - self.config.lambda_value) * l1 + self.config.lambda_value * ld_ssim
        if pointcloud_features is not None and self.config.enable_regularization:
            s = pointcloud_features[point_invalid_mask == 0, 4:7]
            loss = loss + self.config.regularization_weight * torch.norm(torch.exp(s), dim=1).mean()
        return loss, l1, ld_ssim


class _McmcRegulariser(torch.autograd.Function):
    """The terms and their gradient in one launch of ``gsb200_mcmc_regulariser`` on a zero gradient buffer."""

    @staticmethod
    def forward(ctx, features, invalid_mask, lambda_opacity, lambda_scale, num_valid):
        import ctypes
        from . import _lib
        lib = _lib.load()
        feats = features.detach().contiguous()
        grad = torch.zeros_like(feats)
        terms = torch.empty(2, dtype=torch.float32, device=feats.device)
        temp = torch.zeros(int(lib.gsb200_mcmc_temp_bytes()), dtype=torch.uint8, device=feats.device)
        with torch.cuda.device(feats.device):
            stream = torch.cuda.current_stream(feats.device).cuda_stream
            _lib.check(lib.gsb200_mcmc_regulariser(feats.data_ptr(), invalid_mask.data_ptr(), grad.data_ptr(), feats.shape[0],
                                                   int(num_valid), float(lambda_opacity), float(lambda_scale),
                                                   terms.data_ptr(), temp.data_ptr(), ctypes.c_void_p(stream)),
                       "gsb200_mcmc_regulariser")
        ctx.save_for_backward(grad)
        return terms

    @staticmethod
    def backward(ctx, grad_terms):
        (grad,) = ctx.saved_tensors  # columns 4..6 carry the scale term's gradient, column 7 the opacity term's
        scale = torch.cat([grad_terms[1].expand(3), grad_terms[0:1]])
        out = torch.zeros_like(grad)
        out[:, 4:8] = grad[:, 4:8] * scale
        return out, None, None, None, None


def mcmc_regulariser(pointcloud_features: torch.Tensor, point_invalid_mask: torch.Tensor, lambda_opacity: float = 0.01,
                     lambda_scale: float = 0.01, num_valid: Optional[int] = None) -> torch.Tensor:
    """The two L1 regularisers of MCMC densification (``mcmc.py``) as a (2,) tensor {opacity term, scale term}; their sum
    is ``R = lambda_o sum_valid o_i / n_v + lambda_s sum_valid sum_j exp(s_ij) / (3 n_v)`` with o = sigmoid(features[:, 7]),
    s = features[:, 4:7] and n_v the number of rows with ``point_invalid_mask == 0`` (``num_valid``, counted when not
    given; 0 valid rows: both terms 0).  Differentiable in the features.  CUDA float32 tensors run the library's kernel
    (``gsb200_mcmc_regulariser``, sums in double in a fixed order); CPU tensors the torch form, which is the kernel's
    reference."""
    valid = point_invalid_mask == 0
    if num_valid is None:
        num_valid = int(valid.sum())
    if pointcloud_features.is_cuda:
        if pointcloud_features.dtype != torch.float32:
            raise ValueError("the CUDA regulariser takes float32 tensors")
        return _McmcRegulariser.apply(pointcloud_features, point_invalid_mask, lambda_opacity, lambda_scale, num_valid)
    n_v = max(int(num_valid), 1)
    opacity = torch.sigmoid(pointcloud_features[:, 7])[valid].sum() * (lambda_opacity / n_v)
    scale = torch.exp(pointcloud_features[:, 4:7])[valid].sum() * (lambda_scale / (3 * n_v))
    return torch.stack([opacity, scale])
