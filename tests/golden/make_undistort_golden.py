"""Writes undistort_ref.npz: the ten distorted camera sections the project's configurations ship (the eight FAST-LIVO2 scenes, Oxford
Spires and the COLMAP shenzhenbei scene) as data, with what OpenCV makes of them, so that tests compare against OpenCV without cv2:

  cams       [10, 12] float64  model, width, height, fx, fy, cx, cy, d0..d4 (the YAML values)
  new_K      [10, 3, 3] float32  cv2.getOptimalNewCameraMatrix(K, D, size, 0, size, True) with D as set_distortion builds it
  pix        [10, 4096] int32  sampled pixel indices; map1 [10, 4096, 2] int16 and map2 [10, 4096] uint16 the cv2 CV_16SC2 map there
  small_*    one 61x47 model-0 and one 53x41 model-1 camera with a zoomed-out new K: K, D, new K, the full cv2 map, a random
             image and its cv2.remap(INTER_LINEAR)

Run with cv2 4.x: python tests/golden/make_undistort_golden.py"""
import os

import cv2
import numpy as np

LIVO = dict(fx=588.143714607, fy=588.107927227, cx=296.059369138, cy=254.543215481,
            d=(-0.13218037625958456, 0.15360732717073536, 0.00036918417348059815, -0.00031715324469463964, 0.0))
CAMS = [  # name: model, W, H, fx, fy, cx, cy, d0..d4
    ("campus", 0, 640, 512, LIVO["fx"], LIVO["fy"], LIVO["cx"], LIVO["cy"], *LIVO["d"]),
    ("drive", 0, 640, 512, LIVO["fx"], LIVO["fy"], LIVO["cx"], LIVO["cy"], *LIVO["d"]),
    ("cbd", 0, 640, 512, LIVO["fx"], LIVO["fy"], LIVO["cx"], LIVO["cy"], *LIVO["d"]),
    ("culture01", 0, 640, 512, LIVO["fx"], LIVO["fy"], LIVO["cx"], LIVO["cy"], *LIVO["d"]),
    ("station", 0, 640, 512, 646.78472, 646.65775, 313.456795, 261.399612, -0.076160, 0.123001, -0.00113, 0.000251, 0.0),
    ("sysu", 0, 1280, 1024, 1311.89517127580, 1311.36488586115, 656.523841857393, 504.136322840350, -0.0780830982640722,
     0.146382433670493, -0.00110111633050301, -0.00110752991013068, 0.0),
    ("shenzhenbei2", 0, 2048, 1536, 1215.31881774424, 1214.72961288138, 1047.86571859677, 745.068353101898, -0.33574781188503,
     0.10996870793601, 0.000157303079833973, 0.000544930726278493, 0.0),
    ("red_bird", 0, 640, 512, 646.294856087, 646.155780233, 313.423980506, 262.903356268, -0.07581043635239915, 0.1276695531950238,
     -0.0004921162736736936, 3.265638595122261e-05, 0.0),
    ("oxford_spires", 1, 1440, 1080, 698.3946772032825, 698.4629665854908, 718.431814292891, 559.7771701003702, -0.04707469981321094,
     0.011515146787673071, -0.008908394423298474, 0.0018561099343051583, 0.0),
    ("shenzhenbei", 1, 2448, 2048, 1420.341348618206, 1420.997567384703, 1224.37438458383, 1010.762813735306, -0.00425799, 0.00307152,
     -0.0155525, 0.00805682, 0.0),
]


def kmat(fx, fy, cx, cy):
    return np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32)


def cv_map(model, K, D, nK, W, H):
    f = cv2.initUndistortRectifyMap if model == 0 else cv2.fisheye.initUndistortRectifyMap
    return f(K, D, np.eye(3), nK, (W, H), cv2.CV_16SC2)


def main():
    rng = np.random.default_rng(17)
    out = dict(names=np.array([c[0] for c in CAMS]), cams=np.array([c[1:] for c in CAMS], np.float64))
    nks, pix, m1s, m2s = [], [], [], []
    for _, model, W, H, fx, fy, cx, cy, *d in CAMS:
        K = kmat(fx, fy, cx, cy)
        D = np.array([d if model == 0 else d[:4]], np.float32)
        nK = cv2.getOptimalNewCameraMatrix(K, D, (W, H), 0, (W, H), True)[0]
        m1, m2 = cv_map(model, K, D, nK, W, H)
        p = np.sort(rng.choice(W * H, 4096, replace=False)).astype(np.int32)
        nks.append(nK)
        pix.append(p)
        m1s.append(m1.reshape(-1, 2)[p])
        m2s.append(m2.reshape(-1)[p])
    out.update(new_K=np.stack(nks), pix=np.stack(pix), map1=np.stack(m1s), map2=np.stack(m2s))
    for tag, model, W, H, K, D, nK in (
            ("small0", 0, 61, 47, kmat(52.37, 51.91, 30.83, 22.61), np.array([[-0.31, 0.11, 0.0013, -0.0021, -0.017]], np.float32),
             kmat(27.3, 27.1, 29.7, 23.4)),
            ("small1", 1, 53, 41, kmat(30.11, 30.27, 26.3, 20.9), np.array([[-0.047, 0.0115, -0.0089, 0.00186]], np.float32),
             kmat(14.9, 15.2, 26.1, 19.8))):
        m1, m2 = cv_map(model, K, D, nK, W, H)
        img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        out.update({f"{tag}_K": K, f"{tag}_D": D[0], f"{tag}_new_K": nK, f"{tag}_model": np.int32(model), f"{tag}_map1": m1, f"{tag}_map2": m2,
                    f"{tag}_img": img, f"{tag}_remap": cv2.remap(img, m1, m2, cv2.INTER_LINEAR)})
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "undistort_ref.npz"), **out)


if __name__ == "__main__":
    main()
