"""Scene container and on-disk formats either side of the rasteriser (SURVEY §8(f)-4).

``GaussianPointCloudScene`` keeps the reference's surface
(``taichi_3d_gaussian_splatting/GaussianPointCloudScene.py:12-239``): ``nn.Parameter`` ``point_cloud (N,3)``
and ``point_cloud_features (N,56)``, buffers ``point_invalid_mask`` (int8) and ``point_object_id`` (int32),
optional spare capacity (``max_num_points_ratio``), kNN-based initialisation, and the two file formats:

* parquet, columns ``x y z cov_q0-3 cov_s0-2 alpha0 r_sh0-15 g_sh0-15 b_sh0-15`` (:132-146, 183-210);
* the official-3DGS binary PLY ``x y z nx ny nz f_dc_0-2 f_rest_0-44 opacity scale_0-2 rot_0-3``
  (:148-181; import as in ``benchmark/inference_benchmark.py:21-81``): quaternion wxyz on disk <-> xyzw in
  memory, SH stored as DC triple + channel-major rest.

The reference uses the third-party ``plyfile`` package, which is not installed here; the binary
little-endian PLY subset needed (one ``vertex`` element, float32 properties) is read and written directly
with numpy structured arrays.
"""
from dataclasses import dataclass
from typing import Optional, Union

import numpy as np
import torch
import torch.nn as nn

FEATURE_COLUMNS = ([f"cov_q{i}" for i in range(4)] + [f"cov_s{i}" for i in range(3)] + ["alpha0"] +
                   [f"r_sh{i}" for i in range(16)] + [f"g_sh{i}" for i in range(16)] + [f"b_sh{i}" for i in range(16)])
PLY_PROPERTIES = (["x", "y", "z", "nx", "ny", "nz"] + [f"f_dc_{i}" for i in range(3)] +
                  [f"f_rest_{i}" for i in range(45)] + ["opacity"] + [f"scale_{i}" for i in range(3)] +
                  [f"rot_{i}" for i in range(4)])
SH_C0 = 0.28209479177387814


def write_ply_vertices(path: str, columns: dict) -> None:
    """Binary little-endian PLY with one float32 ``vertex`` element; ``columns``: name -> 1-D array."""
    names = list(columns)
    n = len(next(iter(columns.values())))
    rec = np.empty(n, dtype=[(k, "<f4") for k in names])
    for k in names:
        rec[k] = np.asarray(columns[k], dtype=np.float32)
    header = ["ply", "format binary_little_endian 1.0", f"element vertex {n}"]
    header += [f"property float {k}" for k in names] + ["end_header"]
    with open(path, "wb") as f:
        f.write(("\n".join(header) + "\n").encode("ascii"))
        f.write(rec.tobytes())


def read_ply_vertices(path: str) -> dict:
    """Read the ``vertex`` element of a binary little-endian PLY whose properties are scalar."""
    types = {"float": "<f4", "float32": "<f4", "double": "<f8", "float64": "<f8", "uchar": "u1", "uint8": "u1",
             "char": "i1", "int8": "i1", "short": "<i2", "int16": "<i2", "ushort": "<u2", "uint16": "<u2",
             "int": "<i4", "int32": "<i4", "uint": "<u4", "uint32": "<u4"}
    with open(path, "rb") as f:
        if f.readline().strip() != b"ply":
            raise ValueError(f"{path}: not a PLY file")
        fmt, count, props, in_vertex = None, None, [], False
        while True:
            line = f.readline()
            if not line:
                raise ValueError(f"{path}: unterminated PLY header")
            tok = line.decode("ascii").split()
            if not tok:
                continue
            if tok[0] == "format":
                fmt = tok[1]
            elif tok[0] == "element":
                in_vertex = tok[1] == "vertex"
                if in_vertex:
                    if props:
                        raise ValueError(f"{path}: more than one vertex element")
                    count = int(tok[2])
                elif count is None:
                    raise ValueError(f"{path}: the vertex element must come first")
            elif tok[0] == "property" and in_vertex:
                if tok[1] == "list":
                    raise ValueError(f"{path}: list properties are not supported in the vertex element")
                props.append((tok[2], types[tok[1]]))
            elif tok[0] == "end_header":
                break
        if fmt != "binary_little_endian" or count is None:
            raise ValueError(f"{path}: only binary_little_endian PLY with a vertex element is supported")
        data = np.frombuffer(f.read(count * np.dtype(props).itemsize), dtype=props, count=count)
    return {name: np.asarray(data[name]) for name, _ in props}


class GaussianPointCloudScene(nn.Module):
    @dataclass
    class PointCloudSceneConfig:
        # reference: GaussianPointCloudScene.py:14-23
        num_of_features: int = 56
        max_num_points_ratio: Optional[float] = None
        add_sphere: bool = False
        sphere_radius_factor: float = 4.0
        num_points_sphere: int = 10000
        max_initial_covariance: Optional[float] = None
        initial_alpha: float = -2.0
        initial_covariance_ratio: float = 1.0

    def __init__(self, point_cloud: Union[np.ndarray, torch.Tensor], config: "GaussianPointCloudScene.PointCloudSceneConfig",
                 point_cloud_features: Optional[torch.Tensor] = None, point_object_id: Optional[torch.Tensor] = None):
        super().__init__()
        if isinstance(point_cloud, np.ndarray):
            point_cloud = torch.tensor(point_cloud, dtype=torch.float32)  # copies (pandas hands out read-only views)
        point_cloud = torch.as_tensor(point_cloud, dtype=torch.float32)
        if point_cloud.dim() != 2 or point_cloud.shape[1] != 3:
            raise ValueError("point_cloud must be (N, 3)")
        num_points = point_cloud.shape[0]
        capacity = num_points
        if config.max_num_points_ratio is not None:
            capacity = int(num_points * config.max_num_points_ratio)
            if capacity <= num_points:
                raise ValueError("max_num_points_ratio should be greater than 1.0")
        xyz = torch.zeros((capacity, 3), dtype=torch.float32)
        xyz[:num_points] = point_cloud
        feats = torch.zeros((capacity, config.num_of_features), dtype=torch.float32)
        if point_cloud_features is not None:
            feats[:num_points] = torch.as_tensor(point_cloud_features, dtype=torch.float32)
        self.config = config
        self.point_cloud = nn.Parameter(xyz)
        self.point_cloud_features = nn.Parameter(feats)
        invalid = torch.zeros(capacity, dtype=torch.int8)
        invalid[num_points:] = 1
        self.register_buffer("point_invalid_mask", invalid)
        obj = torch.zeros(capacity, dtype=torch.int32)
        if point_object_id is not None:
            obj[:point_object_id.shape[0]] = point_object_id.to(torch.int32)
        self.register_buffer("point_object_id", obj)

    def forward(self):
        return self.point_cloud, self.point_cloud_features

    # GaussianPointCloudScene.py:73-127
    @torch.no_grad()
    def initialize(self, point_cloud_rgb: Optional[np.ndarray] = None, generator: Optional[torch.Generator] = None):
        """Isotropic scale = mean distance to the 3 nearest neighbours, random unit quaternion, fixed opacity logit,
        grey DC colour (or the logit of the given 0..255 RGB divided by the DC basis constant)."""
        from scipy.spatial import cKDTree
        valid = self.point_invalid_mask == 0
        pts = self.point_cloud[valid].detach().cpu().numpy()
        k = min(4, max(pts.shape[0], 1))
        dist, _ = cKDTree(pts).query(pts, k=k)
        dist = np.atleast_2d(dist)
        spread = dist[:, 1:].mean(axis=1) if k > 1 else np.full(pts.shape[0], 1e-6)
        spread = np.clip(spread * self.config.initial_covariance_ratio, 1e-6, self.config.max_initial_covariance)
        f = self.point_cloud_features
        f[valid, 4:7] = torch.tensor(np.log(spread), dtype=torch.float32, device=f.device).unsqueeze(1)
        q = torch.rand(f[:, 0:4].shape, generator=generator).to(f.device)
        f[:, 0:4] = q / q.norm(dim=1, keepdim=True)
        f[:, 7] = self.config.initial_alpha
        f[:, 8:] = 0.0
        f[:, 8] = f[:, 24] = f[:, 40] = 1.0
        if point_cloud_rgb is not None:
            rgb = torch.clamp(torch.as_tensor(point_cloud_rgb, dtype=torch.float32, device=f.device) / 255.0, 0.0, 0.99)
            logit = torch.log(rgb / (1.0 - rgb)) / SH_C0
            for ch, col in enumerate((8, 24, 40)):
                f[valid, col] = logit[:, ch]

    def _valid(self):
        keep = (self.point_invalid_mask == 0).cpu()
        return self.point_cloud.detach().cpu()[keep], self.point_cloud_features.detach().cpu()[keep]

    # GaussianPointCloudScene.py:132-146
    def to_parquet(self, path: str):
        import pandas as pd
        xyz, feat = self._valid()
        frame = pd.concat([pd.DataFrame(xyz.numpy(), columns=["x", "y", "z"]),
                           pd.DataFrame(feat.numpy(), columns=FEATURE_COLUMNS)], axis=1)
        frame.to_parquet(path)

    # GaussianPointCloudScene.py:183-210
    @staticmethod
    def from_parquet(path: str, config: Optional["GaussianPointCloudScene.PointCloudSceneConfig"] = None,
                     generator: Optional[np.random.Generator] = None):
        import pandas as pd
        config = config or GaussianPointCloudScene.PointCloudSceneConfig()
        frame = pd.read_parquet(path)
        if config.add_sphere:
            frame = GaussianPointCloudScene._add_sphere(frame, config.sphere_radius_factor, config.num_points_sphere,
                                                        generator)
        has_rgb = {"r", "g", "b"}.issubset(frame.columns)
        xyz = frame[["x", "y", "z"]].to_numpy()
        if set(FEATURE_COLUMNS).issubset(frame.columns):
            feats = torch.from_numpy(frame[FEATURE_COLUMNS].to_numpy(dtype=np.float32).copy())
            return GaussianPointCloudScene(xyz, config, point_cloud_features=feats)
        scene = GaussianPointCloudScene(xyz, config)
        scene.initialize(point_cloud_rgb=frame[["r", "g", "b"]].to_numpy() if has_rgb else None)
        return scene

    # GaussianPointCloudScene.py:148-181 (official 3DGS layout)
    def to_ply(self, path: str, filter_3d: Optional[torch.Tensor] = None):
        """``filter_3d``: the (N,) 3D smoothing filter of the rows (``mip_filter``; e.g. ``trainer.filter_3d()``), baked into
        ``scale_*`` and ``opacity`` so that any 3DGS viewer shows the filtered scene.  None: the rows as they are."""
        xyz, feat = self._valid()
        if filter_3d is not None:
            from .mip_filter import bake_filter_3d
            keep = (self.point_invalid_mask == 0).cpu()
            feat = bake_filter_3d(feat, filter_3d.detach().cpu()[keep])
        sh = feat[:, 8:].reshape(-1, 3, 16).numpy()
        cols = {"x": xyz[:, 0], "y": xyz[:, 1], "z": xyz[:, 2]}
        for k in ("nx", "ny", "nz"):
            cols[k] = np.zeros(xyz.shape[0], np.float32)
        for ch in range(3):
            cols[f"f_dc_{ch}"] = sh[:, ch, 0]
        rest = sh[:, :, 1:].reshape(-1, 45)  # channel-major: r1..r15 g1..g15 b1..b15
        for i in range(45):
            cols[f"f_rest_{i}"] = rest[:, i]
        cols["opacity"] = feat[:, 7].numpy()
        for i in range(3):
            cols[f"scale_{i}"] = feat[:, 4 + i].numpy()
        for i, src in enumerate((3, 0, 1, 2)):  # xyzw in memory -> wxyz on disk
            cols[f"rot_{i}"] = feat[:, src].numpy()
        write_ply_vertices(path, {k: cols[k] for k in PLY_PROPERTIES})

    # benchmark/inference_benchmark.py:21-81
    @staticmethod
    def from_ply(path: str, config: Optional["GaussianPointCloudScene.PointCloudSceneConfig"] = None):
        config = config or GaussianPointCloudScene.PointCloudSceneConfig()
        v = read_ply_vertices(path)
        n = v["x"].shape[0]
        xyz = np.stack([v["x"], v["y"], v["z"]], axis=1).astype(np.float32)
        rest_names = sorted((k for k in v if k.startswith("f_rest_")), key=lambda s: int(s.split("_")[-1]))
        if len(rest_names) != 45:
            raise ValueError(f"{path}: expected 45 f_rest_* properties (SH degree 3), found {len(rest_names)}")
        rest = np.stack([v[k] for k in rest_names], axis=1).reshape(n, 3, 15)
        rot = np.stack([v[f"rot_{i}"] for i in range(4)], axis=1)
        rot = np.roll(rot, shift=-1, axis=1)  # wxyz -> xyzw
        rot = rot / np.linalg.norm(rot, axis=1, keepdims=True)
        scale = np.stack([v[f"scale_{i}"] for i in range(3)], axis=1)
        feats = np.concatenate(
            [rot, scale, v["opacity"][:, None]] +
            [np.concatenate([v[f"f_dc_{ch}"][:, None], rest[:, ch, :]], axis=1) for ch in range(3)], axis=1)
        return GaussianPointCloudScene(xyz, config, point_cloud_features=torch.from_numpy(feats.astype(np.float32)))

    # GaussianPointCloudScene.py:212-239
    @staticmethod
    def _add_sphere(frame, radius_factor: float, num_points: int, generator: Optional[np.random.Generator] = None):
        """Background shell: points uniform on a sphere of radius (half the largest extent) * radius_factor."""
        import pandas as pd
        rng = generator or np.random.default_rng()
        extent = max(frame[c].max() - frame[c].min() for c in ("x", "y", "z")) / 2.0
        radius = extent * radius_factor
        phi = 2.0 * np.pi * rng.random(num_points)
        theta = np.arccos(2.0 * rng.random(num_points) - 1.0)
        shell = {"x": radius * np.sin(theta) * np.cos(phi), "y": radius * np.sin(theta) * np.sin(phi),
                 "z": radius * np.cos(theta)}
        if {"r", "g", "b"}.issubset(frame.columns):
            for c in ("r", "g", "b"):
                shell[c] = np.full(num_points, 255 // 2, dtype=np.float64)
        return pd.concat([frame, pd.DataFrame(shell)], ignore_index=True)
