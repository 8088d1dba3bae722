"""-m gpu: one ``FusedTrainStep.run`` with the depth, mask, background, feature, appearance and MCMC blocks all on
(``gsb200_train_step_mcmc(t, sup, x, app, mc)``), held to a float64 reference at full frame size and at the narrow and
tiny frames where the per-pixel kernels have edges.

The loss side is recomputed in float64 on the CPU, with torch autograd, from the step's own float32 forward outputs (image,
depth, accumulated alpha, feature map): ``loss.supervision_loss`` around ``_torch_image_loss`` of ``appearance._slice_torch``,
plus ``loss.feature_loss`` and the grid's TV prior.  Against it: the loss outputs, the counts, and the per-pixel gradients
the step hands to the backward (dL/dI, dL/dS, dL/dD, dL/dF) and dL/dG.  The discrete decisions of the reference (the clamp
of the sliced image, the sign of its L1) are the kernel's own: the reference carries the kernel's float32 sliced image as
its forward value and only its gradient in float64, and composites the ground truth in float32 as the kernel does.  Only
the luminance cell and its clamp are decided in float64: pixels within 1e-6 of a z node, 0 or 1 (but not on it) are left
out of dL/dI and dL/dS.

The update side is then replayed in float64 from the kernel's own gradient buffers: Adam on the positions, the 56 feature
columns, the extra features and the visited grid (moments refilled at random, step 10, so that the moments and the bias
corrections decide the update), the MCMC position noise on the post-Adam features, and the MCMC regulariser's gradient on
valid rows behind the camera (whose backward gradient is exactly zero).  Two runs from the same state give bit-identical
loss-side outputs: none of them depends on the backward's float atomics.

Every case first makes a warm-up call with every learning rate 0 (the scene stays as it is, its quaternions normalised).
Then three calls from one state: the targets' exact-tie blocks (depth equal to the rendered depth, mask to the rendered
alpha, feature target to the rendered map, ground truth to the clamped sliced image) are cut from the first one's outputs,
and the other two are compared."""
import functools
import math
from types import SimpleNamespace

import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import CameraInfo
from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR
from taichi_3d_gaussian_splatting_b200.appearance import _slice_torch, bilateral_grid_tv, identity_grids
from taichi_3d_gaussian_splatting_b200.fused_step import FusedTrainStep
from taichi_3d_gaussian_splatting_b200.loss import (SupervisionTargets, _torch_image_loss, feature_loss, mcmc_regulariser,
                                                    supervision_loss)
from taichi_3d_gaussian_splatting_b200.mcmc import MCMCConfig, add_position_noise
from taichi_3d_gaussian_splatting_b200.synthetic import CONFIGS, make_scene

pytestmark = pytest.mark.gpu

N_ROWS = 1_000_003  # 3N and 5N are not multiples of 4: the position and extra-feature Adam steps run their scalar tail
LAMBDA, TV_WEIGHT, FEATURE_WEIGHT = 0.2, 1.0, 0.7
DEPTH_WEIGHT, MASK_WEIGHT = 0.4, 0.3
LR = dict(feature=5e-3, position=2e-4, extra=1e-2, appearance=2e-3)
BETAS, EPS = (0.9, 0.999), 1e-8
STEP = 9  # the step count before the compared call (its Adam step is the 10th)
FOCAL = 1152.0  # C3's 0.6 W; the narrow frames are crops of its image plane
LUMA = (0.299, 0.587, 0.114)
BAND = 1e-6
INT32_MAX = 2 ** 31 - 1

CASES = {
    # name: H, W, depth target, background, feature loss, C, grid (Gx, Gy, Gz), move rows with x > 1 behind the camera
    "A_full_l2": (1072, 1920, "mixed", "random", "l2", 5, (16, 16, 8), False),
    "B_full_ce": (1072, 1920, "none", "black", "cross_entropy", 16, (64, 64, 16), True),
    "C_wide_grid64": (16, 1920, "mixed", "white", "l2", 9, (64, 64, 16), False),
    "C_wide_grid1": (16, 1920, "mixed", "white", "l2", 9, (1, 1, 1), False),
    "C_tall_grid64": (1072, 16, "mixed", "white", "l2", 9, (64, 64, 16), False),
    "C_tall_grid1": (1072, 16, "mixed", "white", "l2", 9, (1, 1, 1), False),
    "D_tiny": (16, 16, "mixed", "random", "l2", 3, (16, 16, 8), False),
    "D_tiny_no_background": (16, 16, "mixed", None, "cross_entropy", 4, (4, 4, 4), False),
}
BACKGROUNDS = {"random": (0.21, 0.83, 0.47), "black": (0.0, 0.0, 0.0), "white": (1.0, 1.0, 1.0)}


class _KernelValue(torch.autograd.Function):
    """The kernel's float32 value ``v`` going forward, ``x``'s gradient going back: the clamp and the L1 sign downstream
    see exactly the values the kernel decided on."""

    @staticmethod
    def forward(ctx, x, v):
        return v.to(x.dtype).clone()

    @staticmethod
    def backward(ctx, grad):
        return grad, None


def _margin(name, err, bar):
    """err / bar (<= 1 passes), printed so that the log shows how close each comparison came."""
    ratio = float(err) / float(bar) if bar > 0 else (0.0 if err == 0 else math.inf)
    print(f"    {name:<34s} err {float(err):.3e}  bar {float(bar):.3e}  ratio {ratio:.3f}")
    return ratio


def _close(name, got, want, rel=1e-5, abs_=1e-6):
    got, want = float(got), float(want)
    assert _margin(name, abs(got - want), rel * abs(want) + abs_) <= 1.0, (name, got, want)


def _close_to_max(name, got, want, keep=None, rel=2e-4):
    got, want = got.double().cpu(), want.double().cpu()
    err = (got - want).abs()
    if keep is not None:
        err = err[keep]
    bar = rel * float(want.abs().max())
    assert float(want.abs().max()) > 0, name
    assert _margin(name, err.max(), bar) <= 1.0, name


# ---------------------------------------------------------------------------------------------- the scene
@functools.lru_cache(maxsize=1)
def _base_rows():
    """C3 padded to N_ROWS rows: invalid rows 0..1999, nearly transparent rows 2000..3999 (the ones the noise's opacity gate
    lets move), and the last 1003 rows (the padding among them) mirrored behind the camera, valid."""
    sc = make_scene(**CONFIGS["C3"])
    n = sc.point_cloud.shape[0]
    pad = N_ROWS - n
    xyz = torch.cat([sc.point_cloud, sc.point_cloud[:pad]]).contiguous()
    feat = torch.cat([sc.point_cloud_features, sc.point_cloud_features[:pad]]).contiguous()
    mask = torch.zeros(N_ROWS, dtype=torch.int8)
    mask[:2000] = 1
    feat[2000:4000, 7] = -6.0
    xyz[-1003:, 2] = -xyz[-1003:, 2]
    return xyz, feat, mask


def _scene(behind_right):
    xyz, feat, mask = (x.clone() for x in _base_rows())
    if behind_right:  # nothing left on the right of the frame: empty pixels, I = 0 and S = 0 exactly
        right = xyz[:, 0] > 1.0
        xyz[right, 2] = -xyz[right, 2].abs()
    return SimpleNamespace(point_cloud=xyz.cuda(), point_cloud_features=feat.cuda(), point_invalid_mask=mask.cuda(),
                           point_object_id=torch.zeros(N_ROWS, dtype=torch.int32, device="cuda"))


def _camera(H, W):
    K = torch.tensor([[FOCAL, 0.0, W / 2.0], [0.0, FOCAL, H / 2.0], [0.0, 0.0, 1.0]], device="cuda")
    return (CameraInfo(K, H, W, 0), torch.tensor([[0.0, 0.0, 0.0, 1.0]], device="cuda"),
            torch.zeros((1, 3), device="cuda"))


def _grids(V, shape, g):
    """Non-identity grids whose affine varies along x, y and, most of all, the luminance axis."""
    gx, gy, gz = shape
    G = identity_grids(V, shape).view(V, 3, 4, gz, gy, gx)
    z = torch.linspace(-0.5, 0.5, gz).view(1, gz, 1, 1)
    for i in range(3):
        G[:, i, i] += 0.3 * z
    G[:, :, 3] += 0.1 * z + 0.05
    G += 0.05 * torch.randn(G.shape, generator=g)
    return G.reshape(V, 12, gz, gy, gx).contiguous().cuda()


# ---------------------------------------------------------------------------------------------- the targets
def _block(H, W, i):
    """The i-th small block of exact ties, away from the others on the larger frames."""
    h, w = max(1, H // 8), max(1, W // 8)
    r0, c0 = (i % 3) * H // 4 + H // 8, (i // 3) * W // 3 + W // 8
    return slice(min(r0, H - h), min(r0, H - h) + h), slice(min(c0, W - w), min(c0, W - w) + w)


def _initial_targets(H, W, depth_kind, kind, C, g):
    gt = torch.rand((3, H, W), generator=g)
    mask = torch.rand((H, W), generator=g)
    mask[::3] = (mask[::3] > 0.5).float()
    depth = 2.0 + 8.0 * torch.rand((H, W), generator=g)
    specials = (0.0, -1.0, float("nan"), float("inf"), -float("inf"))
    if depth_kind == "mixed":
        for k, v in enumerate(specials):
            depth[k::7, (3 * k) % 5::5] = v
    else:  # no valid pixel at all
        for k, v in enumerate(specials):
            depth[k::5] = v
    labels = features = None
    if kind == "cross_entropy":
        labels = torch.randint(-2, C + 3, (H, W), generator=g, dtype=torch.int32)
        labels[0, 0], labels[-1, -1] = -1, C
        labels[1::5, ::3] = INT32_MAX
    else:
        features = torch.randn((H, W, C), generator=g)
        holes = torch.rand((H, W), generator=g) < 0.02
        features[holes, int(torch.randint(0, C, (1,), generator=g))] = float("nan")  # one NaN channel: no target
    cuda = lambda x: None if x is None else x.contiguous().cuda()  # noqa: E731
    return cuda(gt), SupervisionTargets(depth=cuda(depth), mask=cuda(mask), labels=cuda(labels), features=cuda(features))


def _cut_ties(H, W, gt, tg, src, g):
    """The exact-tie blocks, from the outputs ``src`` of a call that renders the same maps as the compared ones, in
    place."""
    b = _block(H, W, 0)
    if ((tg.depth > 0) & torch.isfinite(tg.depth)).any():  # a target with valid pixels: a block equal to the rendered depth
        tg.depth[b] = src.depth[b]
    b = _block(H, W, 1)
    tg.mask[b] = src.acc_alpha[b]
    if tg.features is not None:
        b = _block(H, W, 2)
        tg.features[b] = src.feature_map[b]
    b = _block(H, W, 3)  # L1 ties: mask 1 keeps gt' = gt
    tg.mask[b] = 1.0
    gt[:, b[0], b[1]] = src.sliced_image[b].clamp(0, 1).permute(2, 0, 1)
    # the rest of the ground truth near the render, so that the L1 and SSIM terms are not saturated
    noise = 0.15 * torch.randn(gt.shape, generator=g).to(gt.device)
    noisy = (src.sliced_image.clamp(0, 1).permute(2, 0, 1) + noise).clamp(0, 1)
    keep = torch.ones((H, W), dtype=torch.bool, device=gt.device)
    keep[b] = False
    gt.copy_(torch.where(keep[None], noisy, gt))


# ---------------------------------------------------------------------------------------------- one case
def _outputs(step):
    b = step._last.buffers
    out = dict(image=b.image, depth=b.depth, acc_alpha=b.acc_alpha, feature_map=b.feature_map, sliced_image=b.sliced_image,
               grad_image=b.grad_image, grad_depth=b.grad_depth, grad_alpha=b.grad_alpha, grad_feature_map=b.grad_feature_map,
               grad_grid=step.grad_appearance_grid, loss=step.loss, supervision_loss=step.supervision_loss,
               feature_loss=step.feature_loss, appearance_tv=step.appearance_tv, mcmc_terms=step.mcmc_terms)
    return SimpleNamespace(**{k: v.detach().clone() for k, v in out.items()})


def _run(step, gt, cam, q, t, tg, bg, view, num_valid, lr_scale):
    step.extra_feature_learning_rate = LR["extra"] * lr_scale
    step.appearance_learning_rate = LR["appearance"] * lr_scale
    step.run(gt, q, t, cam, 3, LR["feature"] * lr_scale, LR["position"] * lr_scale, targets=tg, background=bg,
             appearance_view=view, mcmc_num_valid=num_valid)
    torch.cuda.synchronize()
    assert int(step._pinned[step._last.slot][2]) == 0, "the frame overflowed the key capacity"


def _adam64(param, grad, m, v, lr, t):
    """torch's single-tensor Adam in float64."""
    b1, b2 = BETAS
    param, grad, m, v = (x.double() for x in (param, grad, m, v))
    m = m + (grad - m) * (1 - b1)
    v = v * b2 + (1 - b2) * grad * grad
    denom = v.sqrt() / math.sqrt(1 - b2 ** t) + EPS
    return param - (lr / (1 - b1 ** t)) * (m / denom), m, v


def _ulps(x, n=4):
    return n * 2.0 ** -23 * x.abs()


@pytest.mark.parametrize("name", list(CASES))
def test_fused_step_matches_the_float64_reference(name):
    H, W, depth_kind, bg_name, kind, C, grid_shape, behind_right = CASES[name]
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    scene = _scene(behind_right)
    cam, q, t = _camera(H, W)
    scale = 50.0 if kind == "cross_entropy" else 1.0  # logits of +-50
    extra = (scale * (2 * torch.rand((N_ROWS, C), generator=g) - 1)).cuda()
    V, view = 4, 2
    grids = _grids(V, grid_shape, g)
    mc = MCMCConfig(cap_max=N_ROWS, seed=0x1234_5678_9ABC)
    step = FusedTrainStep(scene, GPCR.GaussianPointCloudRasterisationConfig(), LAMBDA, betas=BETAS, eps=EPS,
                          depth_weight=DEPTH_WEIGHT, mask_weight=MASK_WEIGHT, extra_features=extra, feature_loss=kind,
                          feature_weight=FEATURE_WEIGHT, appearance_grids=grids, appearance_tv_weight=TV_WEIGHT, mcmc=mc)
    num_valid = int((scene.point_invalid_mask == 0).sum())
    bg = None if bg_name is None else torch.tensor(BACKGROUNDS[bg_name], device="cuda")
    gt, tg = _initial_targets(H, W, depth_kind, kind, C, g)
    print(f"\n{name}: {H} x {W}, N = {N_ROWS}, {kind} C = {C}, grid {grid_shape}, background {bg_name}")

    # warm-up: every learning rate 0, the scene stays as it is (the quaternions end up normalised in place)
    before = [x.clone() for x in (scene.point_cloud, scene.point_cloud_features[:, 4:], extra, grids)]
    _run(step, gt, cam, q, t, tg, bg, view, num_valid, 0.0)
    for x, x0 in zip((scene.point_cloud, scene.point_cloud_features[:, 4:], extra, grids), before):
        assert torch.equal(x, x0)

    # random moments on the scale of each gradient, step 9 (the compared call is Adam's 10th step)
    gen = torch.Generator(device="cuda").manual_seed(7)
    pairs = [(step.feature_exp_avg, step.feature_exp_avg_sq, step.grad_pointcloud_features),
             (step.position_exp_avg, step.position_exp_avg_sq, step.grad_pointcloud),
             (step.extra_feature_exp_avg, step.extra_feature_exp_avg_sq, step.grad_extra_features),
             (step.appearance_exp_avg[view], step.appearance_exp_avg_sq[view], step.grad_appearance_grid)]
    for m, v, grad in pairs:
        a = max(float(grad.double().pow(2).mean().sqrt()), 1e-12)
        m.copy_(a * (2 * torch.rand(m.shape, generator=gen, device="cuda") - 1))
        v.copy_(a * a * (0.5 + torch.rand(v.shape, generator=gen, device="cuda")))
    tensors = [scene.point_cloud, scene.point_cloud_features, extra, grids] + [x for m, v, _ in pairs for x in (m, v)]
    state0 = [x.clone() for x in tensors]

    # three calls from the same state: the first renders the maps the tie blocks are cut from (a quaternion normalised
    # once may still move by an ulp when normalised again, so the warm-up's maps are not quite these), the other two
    # are compared with each other and with the reference
    runs = []
    for i in range(3):
        for x, x0 in zip(tensors, state0):
            x.copy_(x0)
        step.step_count, step.appearance_steps[view] = STEP, STEP
        _run(step, gt, cam, q, t, tg, bg, view, num_valid, 1.0)
        runs.append(_outputs(step))
        if i == 0:
            _cut_ties(H, W, gt, tg, runs[0], g)
    out = runs[2]
    for key in ("image", "depth", "acc_alpha", "feature_map", "sliced_image"):  # the maps the ties were cut from
        assert torch.equal(getattr(out, key), getattr(runs[0], key)), key
    # bit-identical loss side: nothing of it depends on the backward's float atomics
    for key, a in vars(runs[1]).items():
        assert torch.equal(a, getattr(out, key)), key
    if name == "B_full_ce":
        empty = (out.image == 0).all(-1) & (out.acc_alpha == 0)
        print(f"    empty pixels: {int(empty.sum())}")
        assert int(empty.sum()) > 1000  # luminance exactly 0 on the black background

    _check_loss_side(out, gt, tg, bg, state0[3][view], kind, C, H, W)
    _check_update_side(step, scene, extra, grids, view, state0, pairs, num_valid, mc)


# ---------------------------------------------------------------------------------------------- the loss side
def _check_loss_side(out, gt, tg, bg, grid, kind, C, H, W):
    cpu = lambda x: None if x is None else x.detach().cpu()  # noqa: E731
    I32, D32, S32, F32 = cpu(out.image), cpu(out.depth), cpu(out.acc_alpha), cpu(out.feature_map)
    sliced32, gt32, m32, d32 = cpu(out.sliced_image), cpu(gt), cpu(tg.mask), cpu(tg.depth)
    bg32 = cpu(bg)
    # gt' in float32 with unfused ops: the kernel's own rounding
    gt_p32 = gt32 * m32[None] + (1 - m32)[None] * bg32[:, None, None] if bg32 is not None else gt32

    I = I32.double().requires_grad_(True)
    D = D32.double().requires_grad_(True)
    S = S32.double().requires_grad_(True)
    Fm = F32.double().requires_grad_(True)
    G = cpu(grid).double().requires_grad_(True)
    slice64 = {}

    def image_loss(p, _gt):
        sl = _slice_torch(p, G)
        slice64["value"] = sl.detach()
        slice64["loss"] = _torch_image_loss(_KernelValue.apply(sl, sliced32), gt_p32.double(), LAMBDA)
        return slice64["loss"]

    targets = SupervisionTargets(depth=d32.double(), mask=m32.double())
    total, l1, dssim, mterm, dterm = supervision_loss(I, D, S, gt32.double(), targets,
                                                      None if bg32 is None else bg32.double(), LAMBDA, DEPTH_WEIGHT,
                                                      MASK_WEIGHT, image_loss=image_loss)
    ftargets = SupervisionTargets(labels=cpu(tg.labels), features=None if tg.features is None else cpu(tg.features).double())
    fterm = feature_loss(Fm, ftargets, kind, FEATURE_WEIGHT)
    tv = TV_WEIGHT * bilateral_grid_tv(G)
    (total + fterm + tv).backward()

    # the slice itself, forward
    sl64 = slice64["value"]
    _close_to_max("sliced image (I'')", sliced32, sl64, rel=1e-5)
    # luminance decisions: the exclusion band around 0, 1 and the z nodes
    with torch.no_grad():
        Ip = I32.double() if bg32 is None else I32.double() + (1 - S32.double())[..., None] * bg32.double()
        lum = Ip @ torch.tensor(LUMA, dtype=torch.float64)
        gz = grid.shape[1]
        nodes = torch.unique(torch.cat([torch.linspace(0, 1, gz, dtype=torch.float64), torch.tensor([0.0, 1.0],
                                                                                                     dtype=torch.float64)]))
        dist = (lum[..., None] - nodes).abs().min(-1).values
        band = (dist > 0) & (dist < BAND)
    print(f"    luminance band: {int(band.sum())} of {H * W} pixels; luminance exactly 0: {int((lum == 0).sum())}")
    assert float(band.double().mean()) < 1e-3
    keep = ~band

    # loss outputs
    img_L, img_l1, img_dssim = (float(x.detach()) for x in slice64["loss"])
    _close("L (image loss)", out.loss[0], img_L)
    _close("L1", out.loss[1], img_l1)
    _close("1 - SSIM", out.loss[2], img_dssim)
    _close("supervision total", out.supervision_loss[0], float(total.detach()))
    _close("mask term", out.supervision_loss[1], float(mterm.detach()))
    _close("depth term", out.supervision_loss[2], float(dterm.detach()))
    _close("feature term", out.feature_loss[0], float(fterm.detach()))
    _close("appearance tv", out.appearance_tv[0], float(tv.detach()))
    if kind == "cross_entropy":
        supervised = (tg.labels >= 0) & (tg.labels < C)
    else:
        supervised = torch.isfinite(tg.features).all(-1)
    n_sup = int(supervised.sum())
    assert 0 < n_sup < H * W
    assert float(out.feature_loss[1]) == n_sup

    # dL/dD: exactly float32(+-w / n_valid) or 0
    valid = torch.isfinite(d32) & (d32 > 0)
    n_valid = int(valid.sum())
    scale = torch.tensor(DEPTH_WEIGHT, dtype=torch.float32) / torch.tensor(float(max(n_valid, 1)), dtype=torch.float32)
    e = D32 - d32
    want = torch.where(valid & (e > 0), scale, torch.where(valid & (e < 0), -scale, torch.zeros(())))
    assert torch.equal(cpu(out.grad_depth), want), "dL/dD"
    assert torch.isfinite(out.supervision_loss).all()
    ties = int((valid & (e == 0)).sum())
    print(f"    n_valid {n_valid}, exact depth ties {ties}, n_supervised {n_sup}")
    if n_valid:
        # the count is pinned: a neighbouring count gives another float32 scale
        for other in (n_valid - 1, n_valid + 1):
            assert float(torch.tensor(DEPTH_WEIGHT, dtype=torch.float32) / torch.tensor(float(max(other, 1)))) != float(scale)
        assert ties > 0
    else:
        assert float(out.supervision_loss[2]) == 0.0 and not out.grad_depth.any()

    # dL/dS: with a background against the reference; without one exactly +-w / HW or 0
    e = S32 - m32
    l1_ties = int((sliced32.clamp(0, 1).permute(2, 0, 1) == gt_p32).sum())
    print(f"    exact mask ties {int((e == 0).sum())}, exact L1 ties {l1_ties}")
    assert int((e == 0).sum()) > 0 and l1_ties > 0
    if bg32 is None:
        s = torch.tensor(MASK_WEIGHT, dtype=torch.float32) / torch.tensor(float(H * W), dtype=torch.float32)
        want = torch.where(e > 0, s, torch.where(e < 0, -s, torch.zeros(())))
        assert torch.equal(cpu(out.grad_alpha), want), "dL/dS"
    _close_to_max("dL/dS", out.grad_alpha, S.grad, keep)
    _close_to_max("dL/dI", out.grad_image, I.grad, keep[..., None].expand(H, W, 3))
    _close_to_max("dL/dF", out.grad_feature_map, Fm.grad)
    assert not cpu(out.grad_feature_map)[~cpu(supervised)].any()  # unsupervised pixels: exact zeros
    _close_to_max("dL/dG", out.grad_grid, G.grad)


# ---------------------------------------------------------------------------------------------- the update side
def _check_update_side(step, scene, extra, grids, view, state0, pairs, num_valid, mc):
    t = step.step_count
    assert t == STEP + 1 and step.appearance_steps[view] == STEP + 1
    xyz0, feat0, extra0, grids0 = state0[:4]
    moments0 = state0[4:]
    invalid = scene.point_invalid_mask != 0
    behind = (scene.point_cloud[:, 2] < 0) & ~invalid
    assert int(behind.sum()) >= 1003

    # the MCMC regulariser: its float64 gradient is all a valid row behind the camera gets
    f64 = feat0.double().cpu().requires_grad_(True)
    terms = mcmc_regulariser(f64, scene.point_invalid_mask.cpu(), mc.opacity_reg, mc.scale_reg, num_valid)
    terms.sum().backward()
    _close("mcmc opacity term", step.mcmc_terms[0], float(terms[0]), rel=1e-6, abs_=0.0)
    _close("mcmc scale term", step.mcmc_terms[1], float(terms[1]), rel=1e-6, abs_=0.0)
    gf = step.grad_pointcloud_features
    rb = behind.cpu()
    got, want = gf[behind][:, 4:8].double().cpu(), f64.grad[rb][:, 4:8]
    # 1e-6 relative, and a few float32 roundings of o and 1 - o for the opacity column
    bar = 1e-6 * want.abs() + torch.tensor([0.0, 0.0, 0.0, 1e-7 * mc.opacity_reg / num_valid], dtype=torch.float64)
    assert _margin("regulariser gradient (behind)", ((got - want).abs() / bar).max(), 1.0) <= 1.0
    assert not gf[behind][:, :4].any() and not gf[behind][:, 8:].any()
    assert not gf[invalid].any() and not step.grad_pointcloud[invalid].any()  # invalid rows get nothing

    # Adam, in float64 on the kernel's own gradient buffers
    fm0, fv0, pm0, pv0, em0, ev0, am0, av0 = moments0
    checks = [("features", scene.point_cloud_features, feat0, gf, fm0, fv0, pairs[0], LR["feature"]),
              ("extra features", extra, extra0, step.grad_extra_features, em0, ev0, pairs[2], LR["extra"]),
              ("grid", grids[view], grids0[view], step.grad_appearance_grid, am0, av0, pairs[3], LR["appearance"])]
    for name, param, p0, grad, m0, v0, (m, v, _), lr in checks:
        want, wm, wv = _adam64(p0, grad, m0, v0, lr, t)
        err = (param.double() - want).abs()
        bar = _ulps(want) + 1e-6 * lr
        assert _margin(f"Adam {name}", (err / bar).max(), 1.0) <= 1.0, name
        assert float((param.double() - p0.double()).abs().max()) > 100 * 1e-6 * lr  # the step is not a no-op
        _check_moments(name, m, v, wm, wv, m0, grad)
    # untouched grids of the other views
    others = [i for i in range(grids.shape[0]) if i != view]
    assert torch.equal(grids[others], grids0[others])

    # positions: Adam, then the noise with the post-Adam features the kernel read
    want, wm, wv = _adam64(xyz0, step.grad_pointcloud, pm0, pv0, LR["position"], t)
    adam_only = want.cpu()
    noisy = adam_only.clone()
    feat1 = scene.point_cloud_features.detach().double().cpu()
    noise_scale = mc.noise_lr * LR["position"]
    add_position_noise(noisy, feat1, scene.point_invalid_mask.cpu(), noise_scale, mc.seed, t - 1)
    size = noise_scale * torch.exp(2 * feat1[:, 4:7]).max(1).values * 6.0  # |Sigma| |eps| noise_scale, |eps| < 6
    err = (scene.point_cloud.double().cpu() - noisy).abs()
    bar = _ulps(noisy) + 1e-6 * LR["position"] + 3e-6 * size[:, None] + 1e-12
    assert _margin("Adam + noise positions", (err / bar).max(), 1.0) <= 1.0
    moved = (noisy - adam_only).abs().max(1).values
    print(f"    noise: {int((moved > 1e-6).sum())} rows moved by more than 1e-6, max {float(moved.max()):.3e}")
    assert float(moved.max()) > 1e-4 and not moved[invalid.cpu()].any()
    _check_moments("positions", pairs[1][0], pairs[1][1], wm, wv, pm0, step.grad_pointcloud)


def _check_moments(name, m, v, want_m, want_v, m0, grad):
    """The new moments to a few float32 roundings of their terms (m + (g - m)(1 - b1) may cancel)."""
    bar_m = _ulps(want_m) + _ulps(m0.double()) + _ulps(grad.double()) + 1e-30
    bar_v = _ulps(want_v) + 1e-30
    assert float(((m.double() - want_m).abs() / bar_m).max()) <= 1.0, (name, "exp_avg")
    assert float(((v.double() - want_v).abs() / bar_v).max()) <= 1.0, (name, "exp_avg_sq")
