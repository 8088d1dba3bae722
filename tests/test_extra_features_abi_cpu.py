"""The argument rules of ``gsb200_forward_ext`` / ``gsb200_backward_ext`` and of the operator's ``point_extra_features``,
checked without a device: every rejection comes before any CUDA call."""
import ctypes
import inspect

import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import _lib
from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as G
from taichi_3d_gaussian_splatting_b200.synthetic import make_scene

FAKE = 256  # never dereferenced


def _ext(channels=3, features=FAKE, rasterized=FAKE, grad_rasterized=FAKE, grad_features=FAKE):
    return _lib.GsbExtraFeatureArgs(channels=channels, features=features, rasterized=rasterized,
                                    grad_rasterized=grad_rasterized, grad_features=grad_features)


def test_exports_struct_and_sizes():
    lib = _lib.load()
    for name in ("gsb200_forward_ext", "gsb200_backward_ext"):
        assert name in _lib.EXPORTS and getattr(lib, name).argtypes is not None
    sizes = (ctypes.c_int64 * 7)()
    lib.gsb200_abi_sizes_ext(sizes, 7)
    assert sizes[6] == ctypes.sizeof(_lib.GsbExtraFeatureArgs) == 40


def test_forward_ext_rules():
    lib = _lib.load()
    a = _lib.GsbForwardArgs()
    for ch in (0, -1, 17, 100):
        assert lib.gsb200_forward_ext(ctypes.byref(a), ctypes.byref(_ext(ch))) == -1
        assert b"channels must be in 1..16" in lib.gsb200_last_error()
    for kw in ("features", "rasterized"):
        assert lib.gsb200_forward_ext(ctypes.byref(a), ctypes.byref(_ext(**{kw: None}))) == -1
        assert b"null features / rasterized" in lib.gsb200_last_error()
    rgb = _lib.GsbForwardArgs(rgb_only=1)
    assert lib.gsb200_forward_ext(ctypes.byref(rgb), ctypes.byref(_ext())) == -1
    assert b"rgb_only" in lib.gsb200_last_error()
    # a valid ext reaches the forward's own checks; NULL ext is gsb200_forward
    assert lib.gsb200_forward_ext(ctypes.byref(a), ctypes.byref(_ext())) == -1
    assert b"null camera_intrinsics" in lib.gsb200_last_error()
    assert lib.gsb200_forward_ext(ctypes.byref(a), None) == lib.gsb200_forward(ctypes.byref(a)) == -1
    assert lib.gsb200_forward_ext(None, ctypes.byref(_ext())) == -1
    assert b"args is null" in lib.gsb200_last_error()


def test_backward_ext_rules():
    lib = _lib.load()
    T, K = _lib.GSB_FLAG_BACKWARD_TRANSPOSED, _lib.GSB_FLAG_COMPACT_GRADS
    args = lambda flags: _lib.GsbBackwardArgs(flags=flags)  # noqa: E731
    fake = ctypes.c_void_p(FAKE)
    for ch in (0, 17):
        assert lib.gsb200_backward_ext(ctypes.byref(args(T)), None, None, None, ctypes.byref(_ext(ch))) == -1
        assert b"channels must be in 1..16" in lib.gsb200_last_error()
    for kw in ("features", "grad_rasterized", "grad_features"):
        assert lib.gsb200_backward_ext(ctypes.byref(args(T)), None, None, None, ctypes.byref(_ext(**{kw: None}))) == -1
        assert b"null features / grad_rasterized / grad_features" in lib.gsb200_last_error()
    assert lib.gsb200_backward_ext(ctypes.byref(args(0)), None, None, None, ctypes.byref(_ext())) == -4
    assert b"GSB_FLAG_BACKWARD_TRANSPOSED" in lib.gsb200_last_error()
    assert lib.gsb200_backward_ext(ctypes.byref(args(T | K)), None, None, None, ctypes.byref(_ext())) == -4
    assert b"GSB_FLAG_COMPACT_GRADS" in lib.gsb200_last_error()
    # the depth pair rule of gsb200_backward_aux holds here too
    assert lib.gsb200_backward_ext(ctypes.byref(args(T)), fake, None, None, ctypes.byref(_ext())) == -1
    assert b"both NULL or both set" in lib.gsb200_last_error()
    # a valid ext reaches gsb200_backward's own checks; NULL ext is gsb200_backward_aux
    assert lib.gsb200_backward_ext(ctypes.byref(args(T)), None, None, None, ctypes.byref(_ext())) == -1
    assert b"backward: null pointer argument" in lib.gsb200_last_error()
    for flags in (0, T):
        assert lib.gsb200_backward_ext(ctypes.byref(args(flags)), None, None, None, None) == \
            lib.gsb200_backward_aux(ctypes.byref(args(flags)), None, None, None) == -1
    assert lib.gsb200_backward_ext(None, None, None, None, ctypes.byref(_ext())) == -1
    assert b"args is null" in lib.gsb200_last_error()


def _input(sc):
    return G.GaussianPointCloudRasterisationInput(
        point_cloud=sc.point_cloud, point_cloud_features=sc.point_cloud_features, point_object_id=sc.point_object_id,
        point_invalid_mask=sc.point_invalid_mask, camera_info=sc.camera_info, q_pointcloud_camera=sc.q_pointcloud_camera,
        t_pointcloud_camera=sc.t_pointcloud_camera, color_max_sh_band=3)


class _Exchange:
    world, rank = 2, 0


def test_operator_value_errors():
    Config = G.GaussianPointCloudRasterisationConfig
    param = inspect.signature(G.forward).parameters["point_extra_features"]
    assert param.default is None
    assert "point_extra_features" not in G.GaussianPointCloudRasterisationInput.__dataclass_fields__
    sc = make_scene(50, 32, 32, 0.1, 3, sh_degree=0)
    inp = _input(sc)
    F = torch.zeros((50, 4))
    for op, match in ((G(Config(), backward_impl="butterfly"), "transposed"), (G(Config(rgb_only=True)), "rgb_only"),
                      (G(Config(), gradient_exchange=_Exchange()), "gradient_exchange")):
        with pytest.raises(ValueError, match=match):
            op(inp, point_extra_features=F)
    op = G(Config())
    for bad, match in ((F[:, :0], "1 <= C <= 16"), (torch.zeros((50, 17)), "1 <= C <= 16"), (torch.zeros((49, 4)), "N = 50"),
                       (torch.zeros(50), "N = 50"), (F.double(), "float32"), (torch.zeros((4, 50)).t(), "contiguous"),
                       (F.numpy(), "torch.Tensor")):
        with pytest.raises(ValueError, match=match):
            op(inp, point_extra_features=bad)
    if torch.cuda.is_available():  # the device rule needs a second device type
        with pytest.raises(ValueError, match="must be on"):
            op(inp, point_extra_features=F.cuda())
