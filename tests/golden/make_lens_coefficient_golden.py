"""Writes ``lens_coefficient_vectors.json``: known answers of OpenCV for the coefficient gradient of
``gsb200_backward_lens_grad`` (development tool; the tests read the JSON and do not import cv2).

For each case a camera matrix K (skew-free, as OpenCV takes it), the distortion coefficients and camera-frame points (rvec =
tvec = 0), the pixel positions and the distCoeffs columns of OpenCV's Jacobian, d uv / dk: ``cv2.projectPoints`` (opencv
model, k1 k2 p1 p2 k3: columns 10:15) and ``cv2.fisheye.projectPoints`` (fisheye model, k1..k4: columns 4:8).  The points
include the optical axis and points next to it, where the fisheye helper uses its series.

    python tests/golden/make_lens_coefficient_golden.py
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
    # on the optical axis, a hair off it, and inside the fisheye series' range r^2 < 0.04
    extra = np.array([[0.0, 0.0, 2.0], [1e-7, -2e-7, 3.0], [3e-4, 1e-4, 1.5], [-2e-3, 5e-3, 2.5], [0.2, -0.25, 2.0],
                      [-0.3, 0.1, 1.7]])
    return np.concatenate([extra, pts], 0)


def _opencv(name, K, coeffs, pts):
    uv, jac = cv2.projectPoints(pts.reshape(-1, 1, 3), np.zeros(3), np.zeros(3), K, np.asarray(coeffs, np.float64))
    return dict(name=name, model="opencv", K=K.tolist(), coefficients=list(map(float, coeffs)), points=pts.tolist(),
                uv=uv.reshape(-1, 2).tolist(), duv_dk=jac[:, 10:15].reshape(-1, 2, 5).tolist())


def _fisheye(name, K, coeffs, pts):
    uv, jac = cv2.fisheye.projectPoints(pts.reshape(-1, 1, 3), np.zeros((3, 1)), np.zeros((3, 1)), K,
                                        np.asarray(coeffs, np.float64))
    return dict(name=name, model="fisheye", K=K.tolist(), coefficients=list(map(float, coeffs)) + [0.0], points=pts.tolist(),
                uv=uv.reshape(-1, 2).tolist(), duv_dk=jac[:, 4:8].reshape(-1, 2, 4).tolist())


def main():
    K = np.array([[520.0, 0.0, 330.5], [0.0, 515.0, 241.25], [0.0, 0.0, 1.0]])
    Kw = np.array([[280.0, 0.0, 320.0], [0.0, 280.0, 240.0], [0.0, 0.0, 1.0]])
    cases = [
        _opencv("zero", K, [0.0, 0.0, 0.0, 0.0, 0.0], _points(11, 20, 0.5)),
        _opencv("simple_radial_k1", K, [-0.12, 0.0, 0.0, 0.0, 0.0], _points(12, 20, 0.5)),
        _opencv("opencv_full", K, [-0.21, 0.07, 1.3e-3, -8e-4, -0.012], _points(13, 20, 0.5)),
        _fisheye("fisheye", Kw, [0.05, -0.01, 0.003, -0.0005], _points(14, 20, 1.6)),
        _fisheye("fisheye_strong", Kw, [-0.08, 0.02, -0.004, 0.0002], _points(15, 20, 2.5)),
    ]
    out = dict(cv2_version=cv2.__version__, cases=cases)
    with open(os.path.join(HERE, "lens_coefficient_vectors.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")
    print(f"wrote {len(cases)} cases, cv2 {cv2.__version__}")


if __name__ == "__main__":
    main()
