"""Writes ``lens_vectors.json``: known answers of OpenCV for the lens models of ``gsb200_forward_lens`` (development tool; the
tests read the JSON and do not import cv2).

For each case a camera matrix K (skew-free, as OpenCV takes it), the distortion coefficients and camera-frame points; with
rvec = tvec = 0 the point is given in the camera frame, so the translation columns of OpenCV's Jacobian are d uv / d pc:
``cv2.projectPoints`` (opencv model: columns 3:6) and ``cv2.fisheye.projectPoints`` (fisheye model: columns 11:14).

    python tests/golden/make_lens_golden.py
"""
import json
import os

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def _points(seed, n, spread):
    rng = np.random.default_rng(seed)
    z = rng.uniform(1.0, 6.0, n)
    xy = rng.uniform(-spread, spread, (n, 2)) * z[:, None]
    pts = np.concatenate([xy, z[:, None]], 1)
    # on the optical axis, and a hair off it
    extra = np.array([[0.0, 0.0, 2.0], [1e-7, -2e-7, 3.0], [3e-4, 1e-4, 1.5], [-2e-3, 5e-3, 2.5]])
    return np.concatenate([extra, pts], 0)


def _opencv(name, K, coeffs, pts):
    uv, jac = cv2.projectPoints(pts.reshape(-1, 1, 3), np.zeros(3), np.zeros(3), K, np.asarray(coeffs, np.float64))
    return dict(name=name, model="opencv", K=K.tolist(), coefficients=list(map(float, coeffs)), points=pts.tolist(),
                uv=uv.reshape(-1, 2).tolist(), duv_dpc=jac[:, 3:6].reshape(-1, 2, 3).tolist())


def _fisheye(name, K, coeffs, pts):
    uv, jac = cv2.fisheye.projectPoints(pts.reshape(-1, 1, 3), np.zeros((3, 1)), np.zeros((3, 1)), K,
                                        np.asarray(coeffs, np.float64))
    return dict(name=name, model="fisheye", K=K.tolist(), coefficients=list(map(float, coeffs)) + [0.0], points=pts.tolist(),
                uv=uv.reshape(-1, 2).tolist(), duv_dpc=jac[:, 11:14].reshape(-1, 2, 3).tolist())


def main():
    K = np.array([[520.0, 0.0, 330.5], [0.0, 515.0, 241.25], [0.0, 0.0, 1.0]])
    Kw = np.array([[280.0, 0.0, 320.0], [0.0, 280.0, 240.0], [0.0, 0.0, 1.0]])
    cases = [
        _opencv("simple_radial_k1", K, [-0.12, 0.0, 0.0, 0.0, 0.0], _points(1, 24, 0.5)),
        _opencv("radial_k1_k2", K, [0.08, -0.03, 0.0, 0.0, 0.0], _points(2, 24, 0.55)),
        _opencv("opencv_full", K, [-0.21, 0.07, 1.3e-3, -8e-4, -0.012], _points(3, 24, 0.5)),
        _opencv("strong_barrel", K, [-0.35, 0.12, 0.0, 0.0, -0.02], _points(4, 24, 0.6)),
        _fisheye("fisheye", Kw, [0.05, -0.01, 0.003, -0.0005], _points(5, 24, 1.6)),
        _fisheye("fisheye_strong", Kw, [-0.08, 0.02, -0.004, 0.0002], _points(6, 24, 2.5)),
    ]
    out = dict(cv2_version=cv2.__version__, cases=cases)
    with open(os.path.join(HERE, "lens_vectors.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")
    print(f"wrote {len(cases)} cases, cv2 {cv2.__version__}")


if __name__ == "__main__":
    main()
