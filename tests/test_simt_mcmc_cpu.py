"""The MCMC densification kernels (``csrc/mcmc.cu``) under the SIMT emulator: the position noise against a numpy
re-implementation of Philox4x32-10 + Box-Muller written here from the definition in ``include/gsb200.h``, the regulariser
against torch autograd of ``loss.mcmc_regulariser``, the relocation against a float64 / ``fractions`` evaluation of eq. 9."""
import math
from fractions import Fraction

import numpy as np
import pytest
import torch

from simt_mcmc_helpers import build_mcmc_emulator, emulated_noise, emulated_regulariser, emulated_relocate
from taichi_3d_gaussian_splatting_b200.loss import mcmc_regulariser
from taichi_3d_gaussian_splatting_b200.mcmc import add_position_noise, relocation_opacity_scale


@pytest.fixture(scope="module")
def emu():
    return build_mcmc_emulator()


# ---------------------------------------------------------------------------------------------- the definition, in numpy
def philox4x32_10(c, key):
    c = [np.array(x, np.uint64) for x in c]
    k = [np.uint64(key[0]), np.uint64(key[1])]
    m32 = np.uint64(0xFFFFFFFF)
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c[0]
        p1 = np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k[0], p1 & m32, (p0 >> np.uint64(32)) ^ c[3] ^ k[1], p0 & m32]
        k = [(k[0] + np.uint64(0x9E3779B9)) & m32, (k[1] + np.uint64(0xBB67AE85)) & m32]
    return c


def normals(n, seed, step):
    i = np.arange(n, dtype=np.uint64)
    x = philox4x32_10([i & np.uint64(0xFFFFFFFF), i >> np.uint64(32), np.full(n, step & 0xFFFFFFFF, np.uint64),
                       np.full(n, step >> 32, np.uint64)], (seed & 0xFFFFFFFF, seed >> 32))
    u = [((v >> np.uint64(9)).astype(np.float64) + 0.5) / 2.0 ** 23 for v in x]
    r0, r1 = np.sqrt(-2 * np.log(u[0])), np.sqrt(-2 * np.log(u[2]))
    return np.stack([r0 * np.cos(2 * np.pi * u[1]), r0 * np.sin(2 * np.pi * u[1]), r1 * np.cos(2 * np.pi * u[3])], 1)


def covariance(features):
    f = features.astype(np.float64)
    q = f[:, :4] / np.linalg.norm(f[:, :4], axis=1, keepdims=True)
    x, y, z, w = q.T
    R = np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], 1),
                  np.stack([2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)], 1),
                  np.stack([2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], 1)], 1)
    return R @ (np.exp(2 * f[:, 4:7])[:, :, None] * R.transpose(0, 2, 1))


def expected_noise(features, noise_scale, seed, step, gate_k=100.0, tau=0.005):
    o = 1 / (1 + np.exp(-features[:, 7].astype(np.float64)))
    with np.errstate(over="ignore"):
        gate = 1 / (1 + np.exp(-gate_k * ((1 - o) - (1 - tau))))
    eps = normals(features.shape[0], seed, step)
    return np.einsum("nij,nj->ni", covariance(features), eps) * (noise_scale * gate)[:, None]


def test_philox_known_answers():
    # the Random123 known-answer vectors of philox4x32-10
    assert [int(v) for v in philox4x32_10([0, 0, 0, 0], (0, 0))] == [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]
    ones = 0xFFFFFFFF
    assert [int(v) for v in philox4x32_10([ones] * 4, (ones, ones))] == [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]
    assert [int(v) for v in philox4x32_10([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], (0xa4093822, 0x299f31d0))] == \
        [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1]


def random_rows(n, seed, logit_range=(-7.0, -4.0)):
    rng = np.random.default_rng(seed)
    f = np.zeros((n, 56), np.float32)
    f[:, :4] = rng.normal(size=(n, 4)) * rng.uniform(0.3, 3.0, size=(n, 1))  # unnormalised
    f[:, 4:7] = rng.uniform(-3.0, 0.5, size=(n, 3))
    f[:, 7] = rng.uniform(*logit_range, size=n)
    f[:, 8:] = rng.normal(size=(n, 48))
    xyz = rng.normal(size=(n, 3)).astype(np.float32)
    mask = (rng.uniform(size=n) < 0.2).astype(np.int8)
    return xyz, f, mask


def test_noise_matches_the_definition(emu):
    xyz, f, mask = random_rows(3000, 1)
    seed, step, scale = 0x1234567890ABCDEF, 4321, 0.37
    out = emulated_noise(emu, xyz, f, mask, scale, seed, step)
    want = expected_noise(f, scale, seed, step)
    delta = out.astype(np.float64) - xyz
    valid = mask == 0
    assert np.array_equal(out[~valid], xyz[~valid])  # invalid rows bit-untouched
    # the kernel works in float32: compare at 3e-6 of |Sigma| |eps| noise_scale g (the size of the terms that are summed),
    # plus the rounding of xyz + delta to float32
    o = 1 / (1 + np.exp(-f[:, 7].astype(np.float64)))
    size = scale / (1 + np.exp(-100 * (0.005 - o))) * np.exp(2 * f[:, 4:7].astype(np.float64)).max(1) * \
        np.linalg.norm(normals(len(f), seed, step), axis=1)
    tol = 3e-6 * size[valid, None] + 1.2e-7 * np.abs(xyz[valid]) + 1e-12
    assert np.all(np.abs(delta[valid] - want[valid]) <= tol)
    assert np.abs(want[valid]).max() > 1e-3  # the comparison is not vacuous
    # the torch form of the package draws the same noise
    t_xyz = torch.from_numpy(xyz.copy())
    add_position_noise(t_xyz, torch.from_numpy(f), torch.from_numpy(mask), scale, seed, step)
    assert np.allclose(t_xyz.numpy()[valid] - xyz[valid], want[valid], rtol=1e-3, atol=1e-6)
    assert np.array_equal(t_xyz.numpy()[~valid], xyz[~valid])


def test_noise_is_a_pure_function_of_seed_and_step(emu):
    xyz, f, mask = random_rows(700, 2)
    a = emulated_noise(emu, xyz, f, mask, 1.0, 7, 11)
    assert np.array_equal(a, emulated_noise(emu, xyz, f, mask, 1.0, 7, 11))
    valid = mask == 0
    for seed, step in ((7, 12), (8, 11), (7, 11 + 2 ** 32), (7 + 2 ** 32, 11)):
        b = emulated_noise(emu, xyz, f, mask, 1.0, seed, step)
        assert np.all(np.any(a[valid] != b[valid], axis=1))
    assert np.array_equal(emulated_noise(emu, xyz, f, mask, 1.0, 7, 11, skip=1), xyz)  # the overflow flag: a no-op
    assert np.array_equal(emulated_noise(emu, xyz, f, mask, 1.0, 7, 11, skip=0), a)


def test_the_gate_freezes_opaque_rows(emu):
    f = np.zeros((2, 56), np.float32)
    f[:, 3] = 1.0
    f[0, 7] = math.log(0.9 / 0.1)
    f[1, 7] = math.log(0.001 / 0.999)
    xyz = np.zeros((2, 3), np.float32)
    # the same eps for both rows would need the same counter; compare sizes instead: |row 0| < 1e-30 |row 1|
    out = emulated_noise(emu, xyz, f, np.zeros(2, np.int8), 1.0, 3, 5)
    assert np.abs(out[1]).max() > 1e-3
    assert np.abs(out[0]).max() <= 1e-30 * np.abs(out[1]).max()


def test_noise_statistics(emu):
    n = 120_000
    f = np.zeros((n, 56), np.float32)
    f[:, :4] = (0.3, -0.5, 0.2, 0.7)
    f[:, 4:7] = (-0.2, 0.3, -0.6)
    f[:, 7] = -9.0  # o ~ 1.2e-4: the gate is sigmoid(100 (0.005 - o))
    scale = 0.8
    out = emulated_noise(emu, np.zeros((n, 3), np.float32), f, np.zeros(n, np.int8), scale, 99, 3).astype(np.float64)
    S = covariance(f[:1])[0]
    o = 1 / (1 + math.exp(9.0))
    g = 1 / (1 + math.exp(-100 * (0.005 - o)))
    want = (scale * g) ** 2 * S @ S
    assert np.all(np.abs(out.mean(0)) < 5 * np.sqrt(np.diag(want) / n))
    cov = np.cov(out.T)
    assert np.allclose(cov, want, atol=0.02 * np.abs(want).max())
    eps = np.linalg.solve(S, out.T).T / (scale * g)  # the eps stream itself
    assert np.all(np.abs(eps.mean(0)) < 5 / math.sqrt(n))
    assert np.all(np.abs(eps.var(0) - 1) < 0.02)
    kurt = (eps ** 4).mean(0) / eps.var(0) ** 2
    assert np.all(np.abs(kurt - 3) < 0.1)
    assert np.all(np.abs(np.corrcoef(eps.T) - np.eye(3)) < 0.02)


# ---------------------------------------------------------------------------------------------- regulariser
def test_regulariser_matches_torch_autograd(emu):
    _, f, mask = random_rows(5000, 4, logit_range=(-4.0, 4.0))
    n_v = int((mask == 0).sum())
    rng = np.random.default_rng(5)
    grad0 = rng.normal(size=f.shape).astype(np.float32)
    grad, terms = emulated_regulariser(emu, f, mask, grad0, n_v, 0.01, 0.03)
    ft = torch.from_numpy(f).double().requires_grad_(True)
    want_terms = mcmc_regulariser(ft, torch.from_numpy(mask), 0.01, 0.03)
    want_terms.sum().backward()
    assert np.allclose(terms, want_terms.detach().numpy(), rtol=1e-6)
    added = grad.astype(np.float64) - grad0
    want = ft.grad.numpy()
    assert np.allclose(added, want, rtol=1e-5, atol=2e-7)  # float32 accumulation onto O(1) content
    assert np.abs(want[mask == 0][:, 4:8]).min() > 0
    assert np.array_equal(grad[mask != 0], grad0[mask != 0])  # invalid rows untouched
    assert np.array_equal(grad[:, :4], grad0[:, :4]) and np.array_equal(grad[:, 8:], grad0[:, 8:])
    grad_b, terms_b = emulated_regulariser(emu, f, mask, grad0, n_v, 0.01, 0.03)
    assert np.array_equal(grad, grad_b) and np.array_equal(terms, terms_b)
    # on a zero gradient the result is the plain derivative at float32 accuracy
    grad_z, _ = emulated_regulariser(emu, f, mask, np.zeros_like(f), n_v, 0.01, 0.03)
    assert np.allclose(grad_z, want, rtol=1e-5, atol=0)


def test_regulariser_without_a_valid_row(emu):
    _, f, _ = random_rows(300, 6)
    grad, terms = emulated_regulariser(emu, f, np.ones(300, np.int8), np.ones_like(f), 0, 0.01, 0.01)
    assert np.array_equal(grad, np.ones_like(f)) and np.array_equal(terms, np.zeros(2, np.float32))


# ---------------------------------------------------------------------------------------------- relocation
def reference_D(o_new: float, n: int) -> float:
    """eq. 9's double sum with exact binomials; the alternating sum over k in rationals of the float64 powers."""
    total = 0.0
    for i in range(1, n + 1):
        acc = Fraction(0)
        for k in range(i):
            term = Fraction(math.comb(i - 1, k)) * Fraction(o_new) ** (k + 1) * (-1) ** k
            acc += term * Fraction(1 / math.sqrt(k + 1))
        total += float(acc)
    return total


def one_row_scene(o, n_rows=4):
    f = np.zeros((n_rows, 56), np.float32)
    f[:, 3] = 1.0
    f[:, 4:7] = (-1.0, -0.5, 0.25)
    f[:, 7] = math.log(o / (1 - o))
    f[:, 8:] = np.arange(n_rows * 48, dtype=np.float32).reshape(n_rows, 48)
    return f


def relocated_source(emu, o, count):
    f = one_row_scene(o)
    xyz = np.zeros((4, 3), np.float32)
    emulated_relocate(emu, xyz, f, np.zeros(4, np.int8), np.zeros(4, np.int32), [1], [count], [], [])
    return f


def test_one_copy_is_the_identity(emu):
    for o in (0.006, 0.1, 0.5, 0.9, 0.999):
        before = one_row_scene(o)
        after = relocated_source(emu, o, 0)
        assert np.allclose(after, before, rtol=1e-6, atol=1e-6)
        assert np.array_equal(after[[0, 2, 3]], before[[0, 2, 3]])


@pytest.mark.parametrize("o", [0.006, 0.1, 0.5, 0.9, 0.999])
def test_relocation_arithmetic(emu, o):
    logit = float(np.float32(math.log(o / (1 - o))))
    o = 1 / (1 + math.exp(-logit))  # the opacity the kernel sees
    for n in list(range(2, 52)) + [60, 500]:
        f = relocated_source(emu, o, n - 1)
        n_eff = min(n, 51)
        o_new = 1 / (1 + math.exp(-float(f[1, 7])))
        want_o_new = 1 - (1 - o) ** (1 / n_eff)
        if want_o_new > 0.005:
            assert abs(1 - (1 - o_new) ** n_eff - o) <= 1e-6 * max(1.0, n_eff * o)
        else:
            assert abs(o_new - 0.005) < 1e-8  # clamped to min_opacity
        if n in (2, 3, 7, 20, 51, 500):
            want_shift = math.log(o / reference_D(want_o_new, n_eff))
            shift = f[1, 4:7].astype(np.float64) - one_row_scene(o)[1, 4:7]
            # float32 rounding of s_new; the double sum itself agrees with the rational reference to ~1e-12
            assert np.all(np.abs(shift - want_shift) <= 3e-7 * max(1.0, abs(want_shift)))
            t_logit, t_scale = relocation_opacity_scale(torch.tensor([logit], dtype=torch.float32),
                                                        torch.tensor([[-1.0, -0.5, 0.25]]), torch.tensor([n]))
            assert np.allclose(t_scale.numpy()[0], f[1, 4:7], rtol=0, atol=3e-7)
            assert abs(float(t_logit) - float(f[1, 7])) <= 2e-6 * max(1.0, abs(float(f[1, 7])))


def test_the_double_sum_in_float64_against_rationals():
    # the error statement of the kernel's arithmetic: the float64 evaluation against exact rational accumulation
    worst = 0.0
    for o in (0.006, 0.1, 0.5, 0.9, 0.999):
        for n in (2, 10, 51):
            o_new = 1 - (1 - o) ** (1 / n)
            _, s = relocation_opacity_scale(torch.tensor([math.log(o / (1 - o))], dtype=torch.float64),
                                            torch.zeros((1, 3), dtype=torch.float64), torch.tensor([n]))
            worst = max(worst, abs(float(s[0, 0]) - math.log(o / reference_D(o_new, n))))
    assert worst < 1e-9


@pytest.mark.parametrize("channels", [0, 1, 5, 16])
def test_copies_are_whole_rows_and_moments_are_zeroed(emu, channels):
    rng = np.random.default_rng(channels)
    n = 40
    xyz, f, _ = random_rows(n, 8, logit_range=(-2.0, 2.0))
    mask = np.zeros(n, np.int8)
    mask[30:] = 1
    obj = rng.integers(0, 5, n).astype(np.int32)
    extra = rng.normal(size=(n, channels)).astype(np.float32) if channels else None
    shapes = [(n, 56), (n, 3)] + ([(n, channels)] if channels else [])
    moments = [tuple(rng.normal(size=s).astype(np.float32) for _ in range(2)) for s in shapes]
    before = [tuple(a.copy() for a in pair) for pair in moments]
    f0, xyz0, obj0 = f.copy(), xyz.copy(), obj.copy()
    sources, counts = [2, 5, 9], [1, 3, 1]
    destinations, dest_sources = [30, 12, 31, 14, 39], [5, 2, 5, 9, 5]
    emulated_relocate(emu, xyz, f, mask, obj, sources, counts, destinations, dest_sources, extra=extra, moments=moments)
    touched = sorted(sources + destinations)
    others = [i for i in range(n) if i not in touched]
    for s, k in zip(sources, counts):
        logit, scale = relocation_opacity_scale(torch.from_numpy(f0[s:s + 1, 7]), torch.from_numpy(f0[s:s + 1, 4:7]),
                                                torch.tensor([k + 1]))
        assert np.allclose(f[s, 4:7], scale.numpy()[0], atol=3e-7) and np.isclose(f[s, 7], float(logit), atol=3e-6)
        assert np.array_equal(f[s, :4], f0[s, :4]) and np.array_equal(f[s, 8:], f0[s, 8:])
        assert np.array_equal(xyz[s], xyz0[s]) and mask[s] == 0
    for d, s in zip(destinations, dest_sources):
        assert np.array_equal(f[d], f[s]) and np.array_equal(xyz[d], xyz[s]) and obj[d] == obj[s] and mask[d] == 0
        if channels:
            assert np.array_equal(extra[d], extra[s])
    assert np.array_equal(f[others], f0[others]) and np.array_equal(xyz[others], xyz0[others])
    assert np.array_equal(obj[others], obj0[others])
    assert list(np.nonzero(mask)[0]) == [32, 33, 34, 35, 36, 37, 38]
    for pair, old in zip(moments, before):
        for a, a0 in zip(pair, old):
            assert not a[touched].any() and np.array_equal(a[others], a0[others])


def test_row_ids_outside_the_scene_are_skipped(emu):
    xyz, f, mask = random_rows(8, 9)
    f0, xyz0 = f.copy(), xyz.copy()
    emulated_relocate(emu, xyz, f, mask, np.zeros(8, np.int32), [-1, 8], [1, 1], [3, 9, 2], [8, 1, -2])
    assert np.array_equal(f, f0) and np.array_equal(xyz, xyz0)
