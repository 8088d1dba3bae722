"""Run W warm-up + K measured fwd+bwd steps of the bench workload between cudaProfilerStart/Stop.

    ncu --profile-from-start off --metrics gpu__time_duration.sum --clock-control none --csv \
        --log-file launches.csv python scripts/profile_step.py --steps 2
"""
import argparse, os, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR
from taichi_3d_gaussian_splatting_b200.synthetic import CONFIGS, make_scene

ap = argparse.ArgumentParser()
ap.add_argument("--workload", default="C3")
ap.add_argument("--steps", type=int, default=2)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--forward-only", action="store_true")
a = ap.parse_args()
cfg = CONFIGS[a.workload]
scene = make_scene(**cfg).to("cuda")
scene.point_cloud.requires_grad_(True)
scene.point_cloud_features.requires_grad_(True)
op = GPCR(GPCR.GaussianPointCloudRasterisationConfig())
inp = GPCR.GaussianPointCloudRasterisationInput(
    point_cloud=scene.point_cloud, point_cloud_features=scene.point_cloud_features,
    point_object_id=scene.point_object_id, point_invalid_mask=scene.point_invalid_mask,
    camera_info=scene.camera_info, q_pointcloud_camera=scene.q_pointcloud_camera,
    t_pointcloud_camera=scene.t_pointcloud_camera, color_max_sh_band=3)
g = torch.Generator().manual_seed(1234)
grad_image = torch.randn((cfg["height"], cfg["width"], 3), generator=g).cuda()

def step():
    scene.point_cloud.grad = None
    scene.point_cloud_features.grad = None
    if a.forward_only:
        with torch.no_grad():
            op(inp)
    else:
        image, _, _ = op(inp)
        image.backward(grad_image)

for _ in range(a.warmup):
    step()
torch.cuda.synchronize()
torch.cuda.profiler.start()
for _ in range(a.steps):
    step()
torch.cuda.synchronize()
torch.cuda.profiler.stop()
print("M", op.last_frame.num_points_in_camera, "K", op.last_frame.num_keys)
