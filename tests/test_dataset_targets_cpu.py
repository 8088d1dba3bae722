"""``ImagePoseDataset(path, with_targets=True)``: depth (``.npy``) and mask (an image's last channel) targets cropped and
autoscaled with the image, pixel for pixel; the default items unchanged."""
import json
import os

import numpy as np
import PIL.Image
import pytest
import torch

from taichi_3d_gaussian_splatting_b200.image_pose_dataset import MAX_RESOLUTION_TRAIN, ImagePoseDataset
from taichi_3d_gaussian_splatting_b200.loss import SupervisionTargets

# (height, width): cropped only; cropped only; autoscaled (longest side above MAX_RESOLUTION_TRAIN)
SIZES = [(40, 72), (37, 50), (70, MAX_RESOLUTION_TRAIN + 41)]


def _write(root, sparse=True):
    rng = np.random.default_rng(4)
    records = []
    for i, (h, w) in enumerate(SIZES):
        rgb = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        if i == 1:  # a grey mask file
            mask_file = f"mask{i}.png"
            PIL.Image.fromarray(rgb[:, :, 0], mode="L").save(os.path.join(root, mask_file))
            PIL.Image.fromarray(rgb, mode="RGB").save(os.path.join(root, f"img{i}.png"))
        else:  # an RGBA capture: the alpha channel is the mask, equal to red so that the two can be compared
            rgba = np.concatenate([rgb, rgb[:, :, :1]], axis=2)
            PIL.Image.fromarray(rgba, mode="RGBA").save(os.path.join(root, f"img{i}.png"))
            mask_file = f"img{i}.png"
        # depth = 1 + the pixel's linear index: every target pixel tells which source pixel it came from
        depth = (1.0 + np.arange(h * w, dtype=np.float64).reshape(h, w)).astype(np.float32)
        if sparse and i == 0:
            depth[::2] = 0.0
            depth[1::4, ::3] = np.nan
        np.save(os.path.join(root, f"depth{i}.npy"), depth)
        T = np.eye(4)
        T[:3, 3] = [0.1 * i, -0.2, 0.3]
        records.append(dict(image_path=f"img{i}.png", depth_path=f"depth{i}.npy", mask_path=mask_file,
                            T_pointcloud_camera=T.tolist(), camera_intrinsics=[[100.0, 0, w / 2], [0, 100.0, h / 2], [0, 0, 1]],
                            camera_height=h, camera_width=w, camera_id=i))
    path = os.path.join(root, "train.json")
    with open(path, "w") as f:
        json.dump(records, f)
    return path


@pytest.fixture(scope="module")
def json_path(tmp_path_factory):
    return _write(str(tmp_path_factory.mktemp("posed_targets")))


def test_default_items_are_unchanged_and_targets_come_fifth(json_path):
    plain, with_t = ImagePoseDataset(json_path), ImagePoseDataset(json_path, with_targets=True)
    for i in range(len(SIZES)):
        a, b = plain[i], with_t[i]
        assert len(a) == 4 and len(b) == 5 and isinstance(b[4], SupervisionTargets)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])
        assert torch.equal(a[3].camera_intrinsics, b[3].camera_intrinsics)
        assert (a[3].camera_height, a[3].camera_width) == (b[3].camera_height, b[3].camera_width)


def test_targets_line_up_with_the_cropped_and_scaled_image(json_path):
    ds = ImagePoseDataset(json_path, with_targets=True)
    for i, (h, w) in enumerate(SIZES):
        image, _, _, info, tg = ds[i]
        H, W = info.camera_height, info.camera_width
        assert tg.depth.shape == (H, W) and tg.mask.shape == (H, W)
        assert tg.depth.dtype == tg.mask.dtype == torch.float32 and tg.depth.is_contiguous() and tg.mask.is_contiguous()
        # the mask went through the image's own crop and resize: it equals the red channel it was made from
        assert float((tg.mask - image[0]).abs().max()) <= 1e-6, i
        d = tg.depth.numpy().astype(np.float64)
        if i < 2:  # cropped only: the top-left H x W block of the source, exactly
            src = (1.0 + np.arange(h * w, dtype=np.float64).reshape(h, w))[:H, :W]
            if i == 0:
                src[::2] = 0.0
                src[1::4, ::3] = np.nan
            assert np.array_equal(d, src, equal_nan=True)
        else:  # nearest neighbour: every value is a source pixel, at the place the image's scale maps it to
            idx = d - 1.0
            assert np.array_equal(idx, np.round(idx)) and np.isfinite(idx).all()
            r, c = idx // w, idx % w
            hc = h - h % 16  # the crop comes before the resize
            wc = w - w % 16
            # the resize's own scale (before its crop to the tile multiple), as the intrinsics record it (fx = fy = 100)
            K = info.camera_intrinsics
            ry, rx = 100.0 / float(K[1, 1]), 100.0 / float(K[0, 0])
            ry_, rx_ = (np.arange(H) + 0.5)[:, None] * ry - 0.5, (np.arange(W) + 0.5)[None, :] * rx - 0.5
            assert np.abs(r - ry_).max() <= max(1.0, ry) and np.abs(c - rx_).max() <= max(1.0, rx)
            assert H < hc and W < wc and max(H, W) <= MAX_RESOLUTION_TRAIN


def test_a_target_of_the_wrong_size_is_refused(tmp_path):
    path = _write(str(tmp_path), sparse=False)
    np.save(os.path.join(str(tmp_path), "depth1.npy"), np.ones((SIZES[1][0] + 1, SIZES[1][1]), np.float32))
    ds = ImagePoseDataset(path, with_targets=True)
    ds[0]
    with pytest.raises(ValueError, match="depth"):
        ds[1]
    assert len(ImagePoseDataset(path)[1]) == 4  # without targets nothing is read


def test_records_without_target_keys_give_empty_targets(tmp_path):
    path = _write(str(tmp_path))
    with open(path) as f:
        records = json.load(f)
    del records[0]["depth_path"], records[0]["mask_path"]
    with open(path, "w") as f:
        json.dump(records, f)
    tg = ImagePoseDataset(path, with_targets=True)[0][4]
    assert tg.depth is None and tg.mask is None
