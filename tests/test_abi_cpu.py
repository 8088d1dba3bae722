"""CPU-side checks of the drop-in boundary: the C-ABI library loads without a GPU, exports every symbol
that include/gsb200.h declares, its structs match the ctypes mirrors, the workspace layout arithmetic
is right, and the Python surface keeps the reference's names (SURVEY §8(b)).  No compute calls."""
import dataclasses
import os
import sys
import re

import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    with open(os.path.join(ROOT, "include", "gsb200.h")) as f:
        header = f.read()
    declared = set(re.findall(r"\b(gsb200_[a-z0-9_]+)\s*\(", header))
    assert len(declared) >= 15
    lib = _lib.load()  # also verifies struct sizes against the ctypes mirrors
    for name in sorted(declared):
        assert hasattr(lib, name), f"{name} declared in gsb200.h but not exported by libgsb200.so"
    assert declared == set(_lib.EXPORTS), declared ^ set(_lib.EXPORTS)
    assert lib.gsb200_version() == 102


def test_workspace_layout_arithmetic():
    L = _lib.workspace_layout(1_000_000, 1, 8_000_000, 1072, 1920, 1000.0, 100.0, 0)
    assert (L.key_bytes, L.tile_bits, L.depth_bits, L.radix_bits, L.sort_passes) == (4, 13, 17, 8, 4)  # 8040 tiles, keys <= 1e5
    assert L.scan_blocks == (1_000_000 + 127) // 128  # preprocess CTAs of 128 points
    assert L.key_capacity_padded % 3072 == 0 and L.key_capacity_padded >= 8_000_000  # sort CTAs of 3072 keys
    offs = [L.counters, L.tickets, L.scan_state, L.sort_hist, L.sort_state, L.tile_start, L.tile_end,
            L.poses, L.point_id, L.num_tiles, L.records, L.point_in_camera, L.keys_a, L.keys_b, L.vals_a, L.vals_b, L.keys_c, L.vals_c]
    assert offs == sorted(offs) and all(o % 256 == 0 for o in offs)
    assert L.zero_bytes == L.poses and L.total_bytes > L.vals_c
    # the reference's exact 64-bit packing when asked for, or when the live bits do not fit 32
    L64 = _lib.workspace_layout(1000, 1, 5000, 64, 64, 1000.0, 100.0, _lib.GSB_FLAG_FORCE_KEY64)
    assert (L64.key_bytes, L64.depth_bits) == (8, 32)
    Lbig = _lib.workspace_layout(1000, 1, 5000, 1072, 1920, 2000.0, 1000.0, 0)  # 21 + 13 bits > 32
    assert Lbig.key_bytes == 8
    Ltruck = _lib.workspace_layout(1000, 1, 5000, 544, 976, 2000.0, 10.0, 0)  # Truck YAML: far 2000, scale 10
    assert (Ltruck.key_bytes, Ltruck.depth_bits, Ltruck.tile_bits) == (4, 15, 12)


def test_layout_rejects_bad_sizes():
    with pytest.raises(RuntimeError, match="multiple of the 16x16 tile"):
        _lib.workspace_layout(10, 1, 10, 100, 128, 1000.0, 100.0, 0)
    with pytest.raises(RuntimeError, match="too large"):
        _lib.workspace_layout(1 << 27, 1, 10, 128, 128, 1000.0, 100.0, 0)


def test_python_surface_keeps_reference_names():
    import taichi_3d_gaussian_splatting_b200 as pkg
    from taichi_3d_gaussian_splatting_b200.GaussianPointCloudRasterisation import (
        BOUNDARY_TILES, TILE_HEIGHT, TILE_WIDTH, GaussianPointCloudRasterisation)
    assert (TILE_WIDTH, TILE_HEIGHT, BOUNDARY_TILES) == (16, 16, 3)
    G = GaussianPointCloudRasterisation
    cfg = G.GaussianPointCloudRasterisationConfig()
    assert (cfg.near_plane, cfg.far_plane, cfg.depth_to_sort_key_scale, cfg.rgb_only) == (0.8, 1000.0, 100.0, False)
    # the grad factors are class constants, not dataclass fields (GPCR:782-786)
    assert [f.name for f in dataclasses.fields(cfg)] == ["near_plane", "far_plane", "depth_to_sort_key_scale", "rgb_only"]
    assert (cfg.grad_color_factor, cfg.grad_high_order_color_factor, cfg.grad_s_factor, cfg.grad_q_factor,
            cfg.grad_alpha_factor) == (5.0, 1.0, 0.5, 1.0, 20.0)
    assert [f.name for f in dataclasses.fields(G.GaussianPointCloudRasterisationInput)] == [
        "point_cloud", "point_cloud_features", "point_object_id", "point_invalid_mask", "camera_info",
        "q_pointcloud_camera", "t_pointcloud_camera", "color_max_sh_band"]
    assert [f.name for f in dataclasses.fields(G.BackwardValidPointHookInput)] == [
        "point_id_in_camera_list", "grad_point_in_camera", "grad_pointfeatures_in_camera", "grad_viewspace",
        "magnitude_grad_viewspace", "magnitude_grad_viewspace_on_image", "num_overlap_tiles",
        "num_affected_pixels", "point_depth", "point_uv_in_camera"]
    op = G(cfg)
    assert isinstance(op, torch.nn.Module) and hasattr(op, "_module_function")
    assert pkg.CameraInfo(torch.eye(3), 16, 16, 0).camera_height == 16


def test_operator_refuses_cpu_tensors():
    """The product path must fail loudly without CUDA -- never fall back to the oracle or to PyTorch."""
    from taichi_3d_gaussian_splatting_b200 import CameraInfo, GaussianPointCloudRasterisation as G
    op = G(G.GaussianPointCloudRasterisationConfig())
    inp = G.GaussianPointCloudRasterisationInput(
        point_cloud=torch.zeros(4, 3), point_cloud_features=torch.zeros(4, 56),
        point_object_id=torch.zeros(4, dtype=torch.int32), point_invalid_mask=torch.zeros(4, dtype=torch.int8),
        camera_info=CameraInfo(torch.eye(3), 16, 16, 0), q_pointcloud_camera=torch.tensor([[0., 0, 0, 1]]),
        t_pointcloud_camera=torch.zeros(1, 3))
    with pytest.raises(RuntimeError, match="no CPU path"):
        op(inp)


def test_product_package_never_imports_the_oracle():
    pkg_dir = os.path.join(ROOT, "taichi_3d_gaussian_splatting_b200")
    for dirpath, _, files in os.walk(pkg_dir):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh", ".h")):
                with open(os.path.join(dirpath, fn)) as f:
                    src = f.read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, re.M), f"{fn} imports the oracle"
                assert "gs_oracle" not in src, f"{fn} references the oracle"


def test_fused_l1_has_no_cpu_path_and_reports_its_scratch_size():
    import torch
    from taichi_3d_gaussian_splatting_b200 import fused_l1_loss, fused_l1_loss_with_grad
    lib = _lib.load()
    assert lib.gsb200_l1_loss_temp_bytes() == (4 + 1056) * 4  # ticket block + one partial per CTA (132 SMs x 8)
    a, b = torch.zeros(4, 4, 3), torch.ones(4, 4, 3)
    with pytest.raises(RuntimeError, match="no CPU path"):
        fused_l1_loss_with_grad(a, b)
    with pytest.raises(RuntimeError, match="no CPU path"):
        fused_l1_loss(a.requires_grad_(True), b)
    # argument checks of the C entry point happen before any CUDA call
    assert lib.gsb200_l1_loss(None, None, 0, 0, 1.0, None, None, None, 0, None) == -1
    assert b"l1_loss" in lib.gsb200_last_error()


def test_python_surface_matches_the_reference_modules():
    """tests/golden/surface.json was read off the reference's own modules (dataclass fields with defaults, constructor /
    forward parameters, constants, public methods).  Ours must offer every one of them, with the same defaults; extra
    keyword-only options of ours are allowed."""
    import dataclasses
    import inspect
    import json
    import taichi_3d_gaussian_splatting_b200 as pkg
    mod = sys.modules["taichi_3d_gaussian_splatting_b200.GaussianPointCloudRasterisation"]  # the package re-exports the class under this name
    with open(os.path.join(ROOT, "tests", "golden", "surface.json")) as f:
        ref = json.load(f)
    G, C, S, D = (pkg.GaussianPointCloudRasterisation, pkg.GaussianPointAdaptiveController, pkg.GaussianPointCloudScene,
                  pkg.ImagePoseDataset)

    def check_fields(cls, expected):
        ours = {f.name: f for f in dataclasses.fields(cls)}
        assert [n for n, _, _ in expected] == [n for n in ours if n in {e[0] for e in expected}], cls  # same order
        for name, default, has_default in expected:
            assert name in ours, (cls, name)
            if has_default and not isinstance(default, str):
                assert ours[name].default == default, (cls, name, ours[name].default, default)
            elif not has_default:
                assert ours[name].default is dataclasses.MISSING and ours[name].default_factory is dataclasses.MISSING, (cls, name)

    def check_params(fn, expected):
        ours = [p for p in inspect.signature(fn).parameters if p != "self"]
        assert ours[:len(expected)] == expected, (fn, ours, expected)

    for name, value in ref["constants"].items():
        assert getattr(mod, name) == value
    r = ref["rasterisation"]
    check_fields(G.GaussianPointCloudRasterisationConfig, r["config"])
    check_fields(G.GaussianPointCloudRasterisationInput, r["input"])
    check_fields(G.BackwardValidPointHookInput, r["hook_input"])
    check_params(G.__init__, r["init"])
    check_params(G.forward, r["forward"])
    check_fields(pkg.CameraInfo, ref["camera_info"])
    c = ref["controller"]
    check_fields(C.GaussianPointAdaptiveControllerConfig, c["config"])
    check_fields(C.GaussianPointAdaptiveControllerMaintainedParameters, c["maintained"])
    check_fields(C.GaussianPointAdaptiveControllerDensifyPointInfo, c["densify_info"])
    check_params(C.__init__, c["init"])
    s = ref["scene"]
    check_fields(S.PointCloudSceneConfig, s["config"])
    check_params(S.__init__, s["init"])
    check_params(D.__init__, ref["dataset"]["init"])
    for cls, methods in ((C, c["methods"]), (S, s["methods"]), (D, ref["dataset"]["methods"])):
        for m in methods:
            assert callable(getattr(cls, m)), (cls, m)


def test_fused_image_loss_has_no_cpu_path_and_validates_its_arguments():
    lib = _lib.load()
    from taichi_3d_gaussian_splatting_b200 import fused_image_loss, fused_image_loss_with_grad
    # ticket block, one double per CTA of each kernel (3 channels x 16 x 16 tiles), nine (H-10) x (W-10) derivative planes
    H, W = 544, 976
    tiles_m, tiles_i = ((H - 10 + 15) // 16) * ((W - 10 + 15) // 16), ((H + 15) // 16) * ((W + 15) // 16)
    head = 16 + 8 * 3 * tiles_m + 8 * 3 * tiles_i
    assert lib.gsb200_image_loss_temp_bytes(H, W) == (head + 255) // 256 * 256 + 4 * 9 * (H - 10) * (W - 10)
    assert lib.gsb200_image_loss_temp_bytes(10, 64) == 0  # not larger than the 11-tap window
    a, b = torch.zeros(32, 32, 3), torch.zeros(3, 32, 32)
    with pytest.raises(RuntimeError, match="no CPU path"):
        fused_image_loss_with_grad(a, b)
    with pytest.raises(RuntimeError, match="no CPU path"):
        fused_image_loss(a.requires_grad_(True), b)
    assert lib.gsb200_image_loss(None, None, 32, 32, 0.2, 1.0, None, None, None, 0, None) == -1
    assert b"image_loss" in lib.gsb200_last_error()


def test_load_point_cloud_row_into_gaussian_point_3d():
    """Restated from the reference's tests/GaussianPointCloudRasterisation_test.py:58-99 (same name, arguments, row layout;
    the reference function is a Taichi device function, GPCR:208-236, imported by its controller :4)."""
    from taichi_3d_gaussian_splatting_b200 import load_point_cloud_row_into_gaussian_point_3d
    from taichi_3d_gaussian_splatting_b200.GaussianPointCloudRasterisation import (
        load_point_cloud_row_into_gaussian_point_3d as from_module)
    assert from_module is load_point_cloud_row_into_gaussian_point_3d
    g = torch.Generator().manual_seed(0)
    pointcloud = torch.rand(5, 3, generator=g)
    pointcloud_features = torch.rand(5, 56, generator=g)
    result = load_point_cloud_row_into_gaussian_point_3d(pointcloud=pointcloud, pointcloud_features=pointcloud_features, point_id=2)
    assert torch.equal(result.translation, pointcloud[2])
    assert torch.equal(result.cov_rotation, pointcloud_features[2, :4])
    assert torch.equal(result.cov_scale, pointcloud_features[2, 4:7])
    assert torch.equal(result.alpha, pointcloud_features[2, 7])
    assert torch.equal(result.color_r, pointcloud_features[2, 8:24])
    assert torch.equal(result.color_g, pointcloud_features[2, 24:40])
    assert torch.equal(result.color_b, pointcloud_features[2, 40:56])
