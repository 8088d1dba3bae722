"""Posed-image dataset feeding the operator (SURVEY §8(f)-4, the data format on the caller side of the path).

Same record format and item contract as the reference's ``ImagePoseDataset``
(``taichi_3d_gaussian_splatting/ImagePoseDataset.py:16-103``; format described in ``docs/RawDataFormat.md``):
a JSON list of records with ``image_path``, ``T_pointcloud_camera`` (4x4, camera -> point cloud),
``camera_intrinsics`` (3x3), ``camera_height``, ``camera_width``, ``camera_id``.  ``dataset[i]`` returns
``(image (3,H,W) float32 in [0,1], q_pointcloud_camera (1,4) xyzw, t_pointcloud_camera (1,3), CameraInfo)`` where

* the intrinsics are rescaled from the recorded size to the size of the image actually on disk (:78-83),
* H and W are cropped to multiples of the 16-pixel tile, which the rasteriser requires (:84-88; GPCR:1193-1194),
* frames with a side above ``MAX_RESOLUTION_TRAIN`` are resized (shorter side 1024, longer side capped at 1600,
  antialiased), cropped again and their fx, fy, cx, cy scaled (:41-66).
Records are parsed with ``json`` (no pandas needed); relative image paths are resolved against the JSON file.
With ``with_targets=True`` (an extension) items get a fifth element, ``loss.SupervisionTargets``, from the optional record
keys ``depth_path`` (``.npy`` float32 (H, W) at the resolution of the image on disk, point-cloud units along the optical
axis, 0 or NaN = no measurement) and ``mask_path`` (any image: its last channel / 255, so the alpha of an RGBA file or a
grey mask), cropped and autoscaled with the image: the mask with the image's antialiased resize, the depth with nearest
neighbour so that a sparse map stays sparse.  Two more optional keys carry targets for per-Gaussian feature training:
``labels_path`` (``.npy`` integer (H, W) class ids, read as int32; outside [0, C) = no label) and ``features_path``
(``.npy`` float32 (H, W, C); NaN = no target), both at the resolution of the image on disk and cropped and autoscaled with
the image by nearest neighbour.  The optional key ``loss_weight_path`` gives the view's per-pixel weight of the image loss
(``SupervisionTargets.loss_weight``, 0 = ignore the pixel, e.g. a segmentation mask of people or cars): an image read like
``mask_path`` or a ``.npy`` float32 (H, W), with values in [0, 1], cropped and autoscaled like the mask.
An optional record key ``distortion`` (an extension), ``{"model": "opencv" | "fisheye", "coefficients": [...]}``, gives the
view's ``CameraInfo.distortion`` (``Camera.LensDistortion``).  The coefficients act on the normalised image plane, so
rescaling, cropping and autoscale leave them unchanged.
An optional record key ``rolling_shutter`` (an extension), ``{"linear_velocity": [3], "angular_velocity": [3],
"readout_time": s}``, gives the view's ``CameraInfo.rolling_shutter`` (``Camera.RollingShutter.from_camera_velocity``: the
camera's own velocities in its frame, in scene units/s and rad/s, as visual-inertial odometry reports them, and the sensor's
top-to-bottom readout time).  Row time is normalised by the image height, so rescaling and autoscale keep the motion.
Pinned against the reference class itself: ``tests/golden/make_dataset_golden.py`` imports it (Taichi stubbed) and
stores its outputs for a small generated dataset; ``tests/test_dataset_cpu.py`` compares.
"""
import json
import os
from typing import List, Optional, Tuple

import numpy as np
import torch
import torch.utils.data

from .Camera import CameraInfo, LensDistortion, RollingShutter
from .GaussianPointCloudRasterisation import TILE_HEIGHT, TILE_WIDTH
from .loss import SupervisionTargets
from .utils import SE3_to_quaternion_and_translation_torch

MAX_RESOLUTION_TRAIN = 1600
_REQUIRED = ("image_path", "T_pointcloud_camera", "camera_intrinsics", "camera_height", "camera_width", "camera_id")


def _crop_to_tiles(image: torch.Tensor) -> torch.Tensor:
    h = image.shape[1] - image.shape[1] % TILE_HEIGHT
    w = image.shape[2] - image.shape[2] % TILE_WIDTH
    return image[:3, :h, :w].contiguous()


def _load_image(path: str) -> torch.Tensor:
    """(C,H,W) float32 in [0,1] -- what ``torchvision.transforms.functional.to_tensor`` yields for 8-bit images."""
    import PIL.Image
    with PIL.Image.open(path) as im:
        arr = np.array(im.convert("RGB") if im.mode not in ("RGB", "RGBA", "L") else im)  # writable copy
    if arr.ndim == 2:
        arr = arr[:, :, None]
    return torch.from_numpy(np.ascontiguousarray(arr)).permute(2, 0, 1).to(torch.float32).div(255.0)


class ImagePoseDataset(torch.utils.data.Dataset):
    def __init__(self, dataset_json_path: str, with_targets: bool = False):
        super().__init__()
        self.with_targets = bool(with_targets)
        with open(dataset_json_path) as f:
            self.records: List[dict] = json.load(f)
        self.root = os.path.dirname(os.path.abspath(dataset_json_path))
        for i, rec in enumerate(self.records):
            missing = [k for k in _REQUIRED if k not in rec]
            assert not missing, f"record {i} of {dataset_json_path} lacks {missing}"

    def __len__(self) -> int:
        return len(self.records)

    @staticmethod
    def _autoscale_image_and_camera_info(image: torch.Tensor, camera_info: CameraInfo) -> Tuple[torch.Tensor, CameraInfo]:
        if max(camera_info.camera_height, camera_info.camera_width) <= MAX_RESOLUTION_TRAIN:
            return image, camera_info
        import torchvision.transforms.functional as TF
        resized = TF.resize(image, size=1024, max_size=MAX_RESOLUTION_TRAIN, antialias=True)
        sy = resized.shape[1] / camera_info.camera_height
        sx = resized.shape[2] / camera_info.camera_width
        resized = _crop_to_tiles(resized)
        K = camera_info.camera_intrinsics.clone()
        K[0, 0] *= sx
        K[0, 2] *= sx
        K[1, 1] *= sy
        K[1, 2] *= sy
        return resized, CameraInfo(camera_intrinsics=K, camera_height=resized.shape[1], camera_width=resized.shape[2],
                                   camera_id=camera_info.camera_id, distortion=camera_info.distortion,
                                   rolling_shutter=camera_info.rolling_shutter)

    @staticmethod
    def _distortion(rec: dict) -> Optional[LensDistortion]:
        """The optional record key ``"distortion": {"model": "opencv" | "fisheye", "coefficients": [...]}``."""
        d = rec.get("distortion")
        if d is None:
            return None
        if not isinstance(d, dict) or "model" not in d or "coefficients" not in d:
            raise ValueError(f'"distortion" must be {{"model": ..., "coefficients": [...]}}, got {d!r}')
        return LensDistortion(d["model"], tuple(d["coefficients"]))

    @staticmethod
    def _rolling_shutter(rec: dict) -> Optional[RollingShutter]:
        """The optional record key ``"rolling_shutter": {"linear_velocity": [3], "angular_velocity": [3], "readout_time": s}``."""
        r = rec.get("rolling_shutter")
        if r is None:
            return None
        keys = ("linear_velocity", "angular_velocity", "readout_time")
        if not isinstance(r, dict) or any(k not in r for k in keys):
            raise ValueError(f'"rolling_shutter" must be {{"linear_velocity": [3], "angular_velocity": [3], "readout_time": s}}, '
                             f'got {r!r}')
        if len(r["linear_velocity"]) != 3 or len(r["angular_velocity"]) != 3:
            raise ValueError(f'"rolling_shutter" velocities take 3 values each, got {r!r}')
        return RollingShutter.from_camera_velocity(r["linear_velocity"], r["angular_velocity"], r["readout_time"])

    def _path(self, path: str) -> str:
        if not os.path.isabs(path) and not os.path.exists(path):
            path = os.path.join(self.root, path)
        return path

    def _load_npy(self, rec: dict, key: str, dtype, height: int, width: int, what: str) -> Optional[torch.Tensor]:
        if not rec.get(key):
            return None
        arr = np.load(self._path(rec[key]))
        if dtype == np.int32 and not np.issubdtype(arr.dtype, np.integer):
            raise ValueError(f"{rec[key]}: {what} must be integer, got {arr.dtype}")
        x = torch.from_numpy(np.ascontiguousarray(arr, dtype=dtype))
        if tuple(x.shape[:2]) != (height, width) or x.dim() != (2 if dtype == np.int32 else 3):
            raise ValueError(f"{rec[key]}: {what} is {tuple(x.shape)}, the image is {(height, width)}")
        return x

    def _load_targets(self, rec: dict, height: int, width: int) -> Tuple[torch.Tensor, ...]:
        """(depth, mask, labels, features, loss_weight) at the resolution of the image on disk, or None each: depth, mask
        and loss_weight (H, W) float32, labels (H, W) int32, features (H, W, C) float32."""
        depth = mask = None
        if rec.get("depth_path"):
            depth = torch.from_numpy(np.ascontiguousarray(np.load(self._path(rec["depth_path"])), dtype=np.float32))
            if tuple(depth.shape) != (height, width):
                raise ValueError(f"{rec['depth_path']}: depth map is {tuple(depth.shape)}, the image is {(height, width)}")
        if rec.get("mask_path"):
            m = _load_image(self._path(rec["mask_path"]))
            mask = m[-1].contiguous()
            if tuple(mask.shape) != (height, width):
                raise ValueError(f"{rec['mask_path']}: mask is {tuple(mask.shape)}, the image is {(height, width)}")
        labels = self._load_npy(rec, "labels_path", np.int32, height, width, "label map")
        features = self._load_npy(rec, "features_path", np.float32, height, width, "feature map")
        loss_weight = None
        if rec.get("loss_weight_path"):
            path = self._path(rec["loss_weight_path"])
            if path.endswith(".npy"):
                loss_weight = torch.from_numpy(np.ascontiguousarray(np.load(path), dtype=np.float32))
            else:
                loss_weight = _load_image(path)[-1].contiguous()
            if tuple(loss_weight.shape) != (height, width):
                raise ValueError(f"{rec['loss_weight_path']}: loss weight is {tuple(loss_weight.shape)}, the image is "
                                 f"{(height, width)}")
            if not bool(((loss_weight >= 0) & (loss_weight <= 1)).all()):
                raise ValueError(f"{rec['loss_weight_path']}: loss weights must lie in [0, 1]")
        return depth, mask, labels, features, loss_weight

    @staticmethod
    def _crop_and_scale_nearest(x: torch.Tensor, info: CameraInfo) -> torch.Tensor:
        """(H, W, ...) -> the image's size: cropped to the tile multiple and, if the image was autoscaled, resampled by
        nearest neighbour -- the pixels a nearest-neighbour resize of the image would pick, for any dtype (the pixel indices
        are resized, not the values)."""
        h = x.shape[0] - x.shape[0] % TILE_HEIGHT
        w = x.shape[1] - x.shape[1] % TILE_WIDTH
        x = x[:h, :w]
        if max(h, w) > MAX_RESOLUTION_TRAIN:
            import torchvision.transforms.functional as TF
            idx = torch.arange(h * w, dtype=torch.float64).reshape(1, h, w)
            idx = TF.resize(idx, size=1024, max_size=MAX_RESOLUTION_TRAIN, interpolation=TF.InterpolationMode.NEAREST,
                            antialias=False)
            idx = _crop_to_tiles(idx)[0].long()
            x = x.reshape(h * w, *x.shape[2:])[idx]
        if tuple(x.shape[:2]) != (info.camera_height, info.camera_width):
            raise ValueError(f"target size {tuple(x.shape[:2])} does not match the image's "
                             f"{(info.camera_height, info.camera_width)}")
        return x.contiguous()

    def _crop_and_scale_targets(self, depth, mask, labels, features, loss_weight, info: CameraInfo) -> SupervisionTargets:
        """The targets cropped to the tile multiple and, if the image was autoscaled, resized to its size."""
        out = []
        for x, nearest in ((depth, True), (mask, False), (loss_weight, False)):
            if x is not None:
                x = _crop_to_tiles(x[None])[0]
                if max(x.shape[0], x.shape[1]) > MAX_RESOLUTION_TRAIN:
                    import torchvision.transforms.functional as TF
                    mode = TF.InterpolationMode.NEAREST if nearest else TF.InterpolationMode.BILINEAR
                    x = TF.resize(x[None], size=1024, max_size=MAX_RESOLUTION_TRAIN, interpolation=mode,
                                  antialias=not nearest)
                    x = _crop_to_tiles(x)[0]
                if tuple(x.shape) != (info.camera_height, info.camera_width):
                    raise ValueError(f"target size {tuple(x.shape)} does not match the image's "
                                     f"{(info.camera_height, info.camera_width)}")
                x = x.contiguous()
            out.append(x)
        labels, features = (None if x is None else self._crop_and_scale_nearest(x, info) for x in (labels, features))
        return SupervisionTargets(depth=out[0], mask=out[1], labels=labels, features=features, loss_weight=out[2])

    def __getitem__(self, idx: int):
        rec = self.records[idx]
        path = self._path(rec["image_path"])
        image = _load_image(path)
        T = torch.tensor(rec["T_pointcloud_camera"], dtype=torch.float32).reshape(4, 4)
        q, t = SE3_to_quaternion_and_translation_torch(T.unsqueeze(0))
        K = torch.tensor(rec["camera_intrinsics"], dtype=torch.float32).reshape(3, 3)
        # the image on disk decides the size, not the recorded (COLMAP) one
        K[0, :] = K[0, :] * image.shape[2] / rec["camera_width"]
        K[1, :] = K[1, :] * image.shape[1] / rec["camera_height"]
        if self.with_targets:
            targets = self._load_targets(rec, image.shape[1], image.shape[2])
        image = _crop_to_tiles(image)
        info = CameraInfo(camera_intrinsics=K, camera_height=image.shape[1], camera_width=image.shape[2],
                          camera_id=rec["camera_id"], distortion=self._distortion(rec),
                          rolling_shutter=self._rolling_shutter(rec))
        image, info = self._autoscale_image_and_camera_info(image, info)
        if self.with_targets:
            return image, q, t, info, self._crop_and_scale_targets(*targets, info)
        return image, q, t, info
