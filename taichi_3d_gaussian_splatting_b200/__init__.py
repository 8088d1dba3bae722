"""taichi_3d_gaussian_splatting_b200 -- H100-native (sm_90a) differentiable 3D Gaussian splatting
rasteriser, a drop-in for the hot path of wanmeihuali/taichi_3d_gaussian_splatting
(``GaussianPointCloudRasterisation``).  Host code is Python/PyTorch (memory, streams, autograd,
``torch.distributed``); every kernel is hand-written CUDA behind the C ABI in ``include/gsb200.h``.
"""
from .Camera import CameraInfo, CameraView  # noqa: F401
from .densification import GaussianPointAdaptiveController  # noqa: F401
from .loss import (LossFunction, fused_image_loss, fused_image_loss_with_grad, fused_l1_loss,  # noqa: F401
                   fused_l1_loss_with_grad)
from .optim import FusedAdam  # noqa: F401
from .scene_io import GaussianPointCloudScene  # noqa: F401
from .image_pose_dataset import ImagePoseDataset  # noqa: F401
from .GaussianPointCloudRasterisation import (  # noqa: F401
    BOUNDARY_TILES,
    TILE_HEIGHT,
    TILE_WIDTH,
    GaussianPoint3D,
    GaussianPointCloudRasterisation,
    find_tile_start_and_end,
    load_point_cloud_row_into_gaussian_point_3d,
)

__all__ = ["CameraInfo", "CameraView", "GaussianPointCloudRasterisation", "GaussianPointAdaptiveController",
           "LossFunction", "fused_l1_loss", "fused_l1_loss_with_grad", "fused_image_loss", "fused_image_loss_with_grad", "FusedAdam", "GaussianPointCloudScene", "ImagePoseDataset", "find_tile_start_and_end",
           "load_point_cloud_row_into_gaussian_point_3d", "GaussianPoint3D", "TILE_WIDTH", "TILE_HEIGHT", "BOUNDARY_TILES"]
