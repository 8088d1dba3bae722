"""-m gpu: the autograd inputs of the operator.  On a frozen scene, each camera-parameter tensor and the feature channels,
alone requiring grad, get a gradient of their own shape on their own device, and no other input gets one; a K that requires
grad on an operator without ``differentiable_intrinsics`` leaves the outputs outside the autograd graph."""
import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR
from taichi_3d_gaussian_splatting_b200.Camera import CameraInfo, Defocus, LensDistortion, MotionBlur, RollingShutter
from taichi_3d_gaussian_splatting_b200.synthetic import make_scene

pytestmark = pytest.mark.gpu

Config = GPCR.GaussianPointCloudRasterisationConfig
Input = GPCR.GaussianPointCloudRasterisationInput

_MOTION = ((0.2, -0.05, 0.0), (0.0, 0.03, 0.01))

# (the tensor, the operator option, the camera record it needs, the forward argument it is passed as, its values)
CASES = {
    "point_extra_features": ({}, {}, "point_extra_features", None),
    "camera_intrinsics": ({"differentiable_intrinsics": True}, {}, None, None),
    "q_pointcloud_camera": ({"differentiable_pose": True}, {}, None, None),
    "t_pointcloud_camera": ({"differentiable_pose": True}, {}, None, None),
    "lens_coefficients": ({"differentiable_distortion": True}, {"distortion": LensDistortion("fisheye", (0.1, -0.01, 0.0, 0.0))},
                          "lens_coefficients", [0.1, -0.01, 0.0, 0.0]),
    "rolling_shutter_motion": ({"differentiable_rolling_shutter": True}, {"rolling_shutter": RollingShutter(*_MOTION)},
                               "rolling_shutter_motion", [0.2, -0.05, 0.0, 0.0, 0.03, 0.01]),
    "exposure_motion": ({"differentiable_motion_blur": True}, {"motion_blur": MotionBlur(*_MOTION)}, "exposure_motion",
                        [0.2, -0.05, 0.0, 0.0, 0.03, 0.01]),
    "defocus_parameters": ({"differentiable_defocus": True}, {"defocus": Defocus(0.05, 4.0)}, "defocus_parameters",
                           [0.05, 0.25]),
}


def _inputs(scene, records, K=None):
    sc = scene.to("cuda")
    ci = sc.camera_info
    camera = CameraInfo(ci.camera_intrinsics.clone() if K is None else K, ci.camera_height, ci.camera_width, ci.camera_id,
                        **records)
    return sc, camera


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("device", ["cuda", "cpu"])
def test_each_input_gets_its_gradient_in_its_own_slot(name, device):
    options, records, argument, values = CASES[name]
    if device == "cpu" and values is None:
        pytest.skip("the scene tensors, K and the feature channels live on the scene's device")
    scene = make_scene(4000, 64, 64, 0.05, seed=5, sh_degree=2, yaw_degrees=3.0)
    sc, camera = _inputs(scene, records)
    extra = torch.rand((sc.point_cloud.shape[0], 3), generator=torch.Generator().manual_seed(1)).cuda()
    kwargs = {"point_extra_features": extra}
    tensors = {"point_cloud": sc.point_cloud, "point_cloud_features": sc.point_cloud_features,
               "q_pointcloud_camera": sc.q_pointcloud_camera, "t_pointcloud_camera": sc.t_pointcloud_camera,
               "camera_intrinsics": camera.camera_intrinsics, "point_extra_features": extra}
    if values is not None:
        kwargs[argument] = tensors[argument] = torch.tensor(values, dtype=torch.float32, device=device)
    wanted = tensors[name].requires_grad_(True)
    op = GPCR(Config(), **options)
    outs = op(Input(point_cloud=sc.point_cloud, point_cloud_features=sc.point_cloud_features,
                    point_object_id=sc.point_object_id, point_invalid_mask=sc.point_invalid_mask, camera_info=camera,
                    q_pointcloud_camera=sc.q_pointcloud_camera, t_pointcloud_camera=sc.t_pointcloud_camera,
                    color_max_sh_band=2), **kwargs)
    g = torch.Generator().manual_seed(2)
    loss = (outs[0] * torch.randn(outs[0].shape, generator=g).cuda()).sum() + \
        (outs[-1] * torch.randn(outs[-1].shape, generator=g).cuda()).sum()
    loss.backward()
    assert wanted.grad is not None and wanted.grad.shape == wanted.shape and wanted.grad.device == wanted.device
    assert bool(torch.isfinite(wanted.grad).all())
    for other, t in tensors.items():
        if other != name:
            assert t.grad is None, other


def test_a_K_that_requires_grad_without_differentiable_intrinsics_is_not_an_input():
    scene = make_scene(4000, 64, 64, 0.05, seed=5, sh_degree=2, yaw_degrees=3.0)
    K = scene.camera_info.camera_intrinsics.cuda().requires_grad_(True)
    sc, camera = _inputs(scene, {}, K)
    outs = GPCR(Config())(Input(point_cloud=sc.point_cloud, point_cloud_features=sc.point_cloud_features,
                                point_object_id=sc.point_object_id, point_invalid_mask=sc.point_invalid_mask,
                                camera_info=camera, q_pointcloud_camera=sc.q_pointcloud_camera,
                                t_pointcloud_camera=sc.t_pointcloud_camera, color_max_sh_band=2))
    assert not any(o.requires_grad for o in outs)
