"""``ImagePoseDataset(path, with_targets=True)``: the ``labels_path`` and ``features_path`` targets for per-Gaussian feature
training, read, cropped and autoscaled with the image pixel for pixel (the same pixels as the nearest-neighbour depth)."""
import json
import os

import numpy as np
import PIL.Image
import pytest
import torch

from taichi_3d_gaussian_splatting_b200.image_pose_dataset import MAX_RESOLUTION_TRAIN, ImagePoseDataset

# (height, width): cropped only; autoscaled (longest side above MAX_RESOLUTION_TRAIN)
SIZES = [(40, 72), (70, MAX_RESOLUTION_TRAIN + 41)]
C = 5


def _write(root, label_dtype=np.int64):
    rng = np.random.default_rng(8)
    records = []
    for i, (h, w) in enumerate(SIZES):
        PIL.Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8), mode="RGB").save(os.path.join(root, f"img{i}.png"))
        index = np.arange(h * w, dtype=np.int64).reshape(h, w)  # every target pixel tells which source pixel it came from
        np.save(os.path.join(root, f"depth{i}.npy"), (1.0 + index).astype(np.float32))
        labels = index.astype(label_dtype)
        labels[0, :3] = [-1, 2147483647, -2147483648]  # "no label" values survive exactly
        np.save(os.path.join(root, f"labels{i}.npy"), labels)
        features = np.stack([index * (k + 1) % 9973 - 0.5 * k for k in range(C)], axis=-1).astype(np.float32)
        features[1, 1, 2] = np.nan
        np.save(os.path.join(root, f"features{i}.npy"), features)
        records.append(dict(image_path=f"img{i}.png", depth_path=f"depth{i}.npy", labels_path=f"labels{i}.npy",
                            features_path=f"features{i}.npy", T_pointcloud_camera=np.eye(4).tolist(),
                            camera_intrinsics=[[100.0, 0, w / 2], [0, 100.0, h / 2], [0, 0, 1]], camera_height=h,
                            camera_width=w, camera_id=i))
    path = os.path.join(root, "train.json")
    with open(path, "w") as f:
        json.dump(records, f)
    return path


@pytest.fixture(scope="module")
def json_path(tmp_path_factory):
    return _write(str(tmp_path_factory.mktemp("posed_feature_targets")))


def test_labels_and_features_line_up_with_the_nearest_neighbour_depth(json_path):
    ds = ImagePoseDataset(json_path, with_targets=True)
    for i, (h, w) in enumerate(SIZES):
        image, _, _, info, tg = ds[i]
        H, W = info.camera_height, info.camera_width
        assert tg.labels.shape == (H, W) and tg.labels.dtype == torch.int32 and tg.labels.is_contiguous()
        assert tg.features.shape == (H, W, C) and tg.features.dtype == torch.float32 and tg.features.is_contiguous()
        src = (tg.depth.numpy().astype(np.float64) - 1.0).astype(np.int64)  # the source pixel of every target pixel
        labels = np.arange(h * w, dtype=np.int64)
        labels[:3] = [-1, 2147483647, -2147483648]
        assert np.array_equal(tg.labels.numpy(), labels[src].astype(np.int32)), i
        index = np.arange(h * w, dtype=np.int64)
        feats = np.stack([index * (k + 1) % 9973 - 0.5 * k for k in range(C)], axis=-1).astype(np.float32)
        feats[1 * w + 1, 2] = np.nan
        assert np.array_equal(tg.features.numpy(), feats[src], equal_nan=True), i
        if i == 0:  # cropped only: the top-left block
            assert (H, W) == (h - h % 16, w - w % 16) and np.array_equal(src, index.reshape(h, w)[:H, :W])
        else:
            assert max(H, W) <= MAX_RESOLUTION_TRAIN < w


def test_int32_label_files_are_read_as_they_are(tmp_path):
    ds = ImagePoseDataset(_write(str(tmp_path), label_dtype=np.int32), with_targets=True)
    tg = ds[0][4]
    assert tg.labels.dtype == torch.int32 and int(tg.labels[0, 1]) == 2147483647 and int(tg.labels[0, 2]) == -2147483648


@pytest.mark.parametrize("key,bad", [("labels", np.zeros((41, 72), np.int32)), ("labels", np.zeros((40, 72), np.float32)),
                                     ("labels", np.zeros((40, 72, 1), np.int32)), ("features", np.zeros((40, 71, C), np.float32)),
                                     ("features", np.zeros((40, 72), np.float32))])
def test_a_label_or_feature_map_of_the_wrong_shape_or_type_is_refused(tmp_path, key, bad):
    path = _write(str(tmp_path))
    np.save(os.path.join(str(tmp_path), f"{key}0.npy"), bad)
    ds = ImagePoseDataset(path, with_targets=True)
    with pytest.raises(ValueError, match="label map" if key == "labels" else "feature map"):
        ds[0]
    ds[1]
    assert len(ImagePoseDataset(path)[0]) == 4  # without targets nothing is read


def test_records_without_the_keys_give_no_label_or_feature_targets(tmp_path):
    path = _write(str(tmp_path))
    with open(path) as f:
        records = json.load(f)
    del records[0]["labels_path"], records[0]["features_path"]
    with open(path, "w") as f:
        json.dump(records, f)
    tg = ImagePoseDataset(path, with_targets=True)[0][4]
    assert tg.labels is None and tg.features is None and tg.depth is not None
