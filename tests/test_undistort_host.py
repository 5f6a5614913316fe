"""Undistortion of distorted cameras (DESIGN 7r) without a GPU: the numpy restatements of gssdf_undistort_map and gssdf_undistort_u8
(undistort_oracle.py) and cameras.optimal_new_camera_matrix against OpenCV (cv2 when it imports, else the goldens it wrote), the
config and cameras.txt semantics of sensor::Cameras, and the argument errors of the new entry points."""
import ctypes
import os

import numpy as np
import pytest
import torch

import undistort_oracle as U
from gssdf_b200 import cameras as CM

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "undistort_ref.npz"))


def _K(fx, fy, cx, cy):
    return np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32)


def shipped():
    """(name, model, W, H, K, D) of the ten shipped camera sections, D as set_distortion builds it"""
    for name, c in zip(GOLD["names"], GOLD["cams"]):
        model, W, H = int(c[0]), int(c[1]), int(c[2])
        d = np.array(c[7:12], np.float32)
        yield str(name), model, W, H, _K(*c[3:7]), d if model == 0 else d[:4]


def random_cameras(n, seed):
    rng = np.random.default_rng(seed)
    for k in range(n):
        W, H = int(rng.integers(2, 160)), int(rng.integers(2, 130))
        f = rng.uniform(0.4, 1.6) * max(W, H)
        model = k % 2
        d = rng.normal(0, [0.12, 0.05, 0.002, 0.002, 0.01]) if model == 0 else rng.normal(0, [0.05, 0.02, 0.01, 0.003])
        K = _K(f * rng.uniform(0.95, 1.05), f * rng.uniform(0.95, 1.05), W / 2 * rng.uniform(0.9, 1.1), H / 2 * rng.uniform(0.9, 1.1))
        yield model, W, H, K, d.astype(np.float32)


def test_goldens_match_the_restatements():
    """No cv2 needed: the new K of every shipped camera, the sampled map entries and the small maps and remaps."""
    for i, (name, model, W, H, K, d) in enumerate(shipped()):
        nK = CM.optimal_new_camera_matrix(K, d, W, H)
        assert np.array_equal(nK, GOLD["new_K"][i]), name
        m = U.undistort_map(K, d, nK, model, W, H).reshape(-1, 4)[GOLD["pix"][i]]
        assert np.array_equal(m[:, :2], GOLD["map1"][i]) and np.array_equal(m[:, 2].astype(np.uint16), GOLD["map2"][i]), name
    for tag in ("small0", "small1"):
        H, W = GOLD[f"{tag}_img"].shape[:2]
        m = U.undistort_map(GOLD[f"{tag}_K"], GOLD[f"{tag}_D"], GOLD[f"{tag}_new_K"], int(GOLD[f"{tag}_model"]), W, H)
        assert np.array_equal(m[..., :2], GOLD[f"{tag}_map1"]) and np.array_equal(m[..., 2].astype(np.uint16), GOLD[f"{tag}_map2"]), tag
        assert (m[..., 3] == 0).all()
        assert np.array_equal(U.remap(GOLD[f"{tag}_img"], m), GOLD[f"{tag}_remap"]), tag


def _cv_maps(cv2, model, K, d, nK, W, H):
    f = cv2.initUndistortRectifyMap if model == 0 else cv2.fisheye.initUndistortRectifyMap
    return f(K, d.reshape(1, -1), np.eye(3), nK, (W, H), cv2.CV_16SC2)


def _same_map(m, m1, m2):
    return np.array_equal(m[..., :2], m1) and np.array_equal(m[..., 2].astype(np.uint16), m2)


def test_restatements_equal_cv2_on_shipped_and_random_cameras():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(5)
    cams = [(model, W, H, K, d) for _, model, W, H, K, d in shipped()] + list(random_cameras(240, 11))
    for n, (model, W, H, K, d) in enumerate(cams):
        nK = cv2.getOptimalNewCameraMatrix(K, d.reshape(1, -1), (W, H), 0, (W, H), True)[0]
        assert np.array_equal(CM.optimal_new_camera_matrix(K, d, W, H), nK), (n, W, H)
        m1, m2 = _cv_maps(cv2, model, K, d, nK, W, H)
        m = U.undistort_map(K, d, nK, model, W, H)
        assert _same_map(m, m1, m2), (n, model, W, H)
        if n < 10 and W * H > 1_000_000:
            continue  # the remap of the big shipped frames is covered by the random ones
        img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        assert np.array_equal(U.remap(img, m), cv2.remap(img, m1, m2, cv2.INTER_LINEAR)), (n, model, W, H)


def test_zoomed_out_new_K_exercises_the_border():
    """An explicit new K at half the focal length: much of the output maps outside the source frame, partly outside and wholly outside
    the 2x2 blocks, and a textured frame remaps byte for byte."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(3)
    for model, d in ((0, np.array([-0.31, 0.11, 0.0013, -0.0021, -0.017], np.float32)),
                     (1, np.array([-0.047, 0.0115, -0.0089, 0.00186], np.float32))):
        W, H = 333, 251
        K, nK = _K(301.37, 299.83, 170.21, 122.77), _K(151.3, 150.9, 166.4, 125.1)
        m1, m2 = _cv_maps(cv2, model, K, d, nK, W, H)
        m = U.undistort_map(K, d, nK, model, W, H)
        assert _same_map(m, m1, m2)
        sx, sy = m[..., 0].astype(int), m[..., 1].astype(int)
        outside = (sx >= W) | (sx + 1 < 0) | (sy >= H) | (sy + 1 < 0)
        partial = ~outside & ((sx < 0) | (sx + 1 >= W) | (sy < 0) | (sy + 1 >= H))
        assert outside.sum() > 1000 and partial.sum() > 100
        img = rng.integers(1, 256, (H, W, 3), dtype=np.uint8)
        got = U.remap(img, m)
        assert np.array_equal(got, cv2.remap(img, m1, m2, cv2.INTER_LINEAR))
        assert (got[outside] == 0).all()


def test_camera_from_config_follows_set_distortion():
    cv2 = pytest.importorskip("cv2")
    # campus.yaml
    c = CM.camera_from_config(0, 640, 512, 588.143714607, 588.107927227, 296.059369138, 254.543215481, -0.13218037625958456,
                              0.15360732717073536, 0.00036918417348059815, -0.00031715324469463964, 0.0)
    K = _K(588.143714607, 588.107927227, 296.059369138, 254.543215481)
    D = np.array([[-0.13218037625958456, 0.15360732717073536, 0.00036918417348059815, -0.00031715324469463964, 0.0]], np.float32)
    nK = cv2.getOptimalNewCameraMatrix(K, D, (640, 512), 0, (640, 512), True)[0]
    assert (c.W, c.H) == (640, 512) and np.array_equal(c.K.numpy(), nK) and c.undistortion.model == 0
    assert np.array_equal(c.undistortion.d, D[0]) and (c.undistortion.W, c.undistortion.H) == (640, 512)
    # a model-1 section: the new K reads d0..d3 as k1 k2 p1 p2, the map as the fisheye k1..k4; scale applies after, to size and K
    args = (1, 1440, 1080, 698.3946772032825, 698.4629665854908, 718.431814292891, 559.7771701003702, -0.04707469981321094,
            0.011515146787673071, -0.008908394423298474, 0.0018561099343051583, 0.0)
    c = CM.camera_from_config(*args, scale=0.5)
    K = _K(*args[3:7])
    D4 = np.array([args[7:11]], np.float32)
    nK = cv2.getOptimalNewCameraMatrix(K, D4, (1440, 1080), 0, (1440, 1080), True)[0]
    s = np.float32(0.5)
    assert (c.W, c.H) == (720, 540)
    assert np.array_equal(c.K.numpy(), np.array([[s * nK[0, 0], 0, s * nK[0, 2]], [0, s * nK[1, 1], s * nK[1, 2]], [0, 0, 1]], np.float32))
    u = c.undistortion
    assert (u.W, u.H, u.model) == (1440, 1080, 1) and np.array_equal(u.d, D4[0]) and np.array_equal(u.K.numpy(), nK)
    # no d0: pinhole, scaled
    c = CM.camera_from_config(0, 641, 479, 500.5, 501.25, 320.1, 239.7, scale=0.3)
    s = np.float32(0.3)
    assert c.undistortion is None and (c.W, c.H) == (int(s * np.float32(641)), int(s * np.float32(479)))
    assert np.array_equal(c.K.numpy(), np.array([[s * np.float32(500.5), 0, s * np.float32(320.1)], [0, s * np.float32(501.25),
                                                                                                        s * np.float32(239.7)], [0, 0, 1]], np.float32))
    with pytest.raises(ValueError):
        CM.camera_from_config(2, 64, 48, 50, 50, 32, 24, 0.1)


def test_read_colmap_cameras(tmp_path):
    cv2 = pytest.importorskip("cv2")
    from gssdf_b200 import io as IO
    txt = ("# cameras\n1 PINHOLE 1920 1080 1371.7 1371.7 960 540\n2 OPENCV 1279 719 903.3333 901.15 639.7 359.1 -0.05 0.01 0.001 -0.0002\n"
           "3 OPENCV_FISHEYE 2448 2048 1420.341348618206 1420.997567384703 1224.37438458383 1010.762813735306 -0.00425799 0.00307152 "
           "-0.0155525 0.00805682\n")
    p = tmp_path / "cameras.txt"
    p.write_text(txt)
    (tmp_path / "pin.txt").write_text("\n".join(txt.split("\n")[:3]))
    for scale in (1.0, 0.5):
        cams = CM.read_colmap_cameras(str(p), scale)
        pin = IO.load_colmap_cameras(str(tmp_path / "pin.txt"), scale)
        for i in (1, 2):  # pinhole lines read exactly as io.load_colmap_cameras reads them
            assert (cams[i].W, cams[i].H) == pin[i][:2] and torch.equal(cams[i].K, pin[i][2]) and cams[i].undistortion is None
        u = cams[3].undistortion
        K = _K(*[np.float32(v) for v in (1420.341348618206, 1420.997567384703, 1224.37438458383, 1010.762813735306)])
        D = np.array([[-0.00425799, 0.00307152, -0.0155525, 0.00805682]], np.float32)
        nK = cv2.getOptimalNewCameraMatrix(K, D, (2448, 2048), 0, (2448, 2048), True)[0]
        s = np.float32(scale)
        assert (u.W, u.H, u.model) == (2448, 2048, 1) and np.array_equal(u.K.numpy(), nK) and np.array_equal(u.d, D[0])
        assert (cams[3].W, cams[3].H) == (int(s * np.float32(2448)), int(s * np.float32(2048)))
        assert np.array_equal(cams[3].K.numpy()[[0, 1, 0, 1], [0, 1, 2, 2]], s * nK[[0, 1, 0, 1], [0, 1, 2, 2]])
    with pytest.raises(ValueError):
        IO.load_colmap_cameras(str(p))  # unchanged: the pinhole reader still refuses fisheye lines
    (tmp_path / "bad.txt").write_text("4 OPENCV_FISHEYE 64 48 50 50 32 24 0.1 0.2\n")
    with pytest.raises(ValueError):
        CM.read_colmap_cameras(str(tmp_path / "bad.txt"))
    (tmp_path / "bad2.txt").write_text("4 SIMPLE_RADIAL 64 48 50 32 24 0.1\n")
    with pytest.raises(ValueError):
        CM.read_colmap_cameras(str(tmp_path / "bad2.txt"))


def test_undistort_frames_argument_errors():
    u = CM.Undistortion(8, 6, _K(10, 10, 4, 3), [0.1, 0.0, 0.0, 0.0, 0.0], 0, device="cpu")
    with pytest.raises(ValueError):
        CM.undistort_frames(torch.zeros(2, 6, 8, 3), u)  # not uint8
    with pytest.raises(ValueError):
        CM.undistort_frames(torch.zeros(2, 7, 8, 3, dtype=torch.uint8), u)  # size differs from the camera's
    with pytest.raises(ValueError):
        CM.undistort_frames(torch.zeros(2, 6, 8, 3, dtype=torch.uint8), [u], camera_ids=[0, 1])
    with pytest.raises(ValueError, match="not an Undistortion"):
        CM.undistort_frames(torch.zeros(2, 6, 8, 3, dtype=torch.uint8), [u, None], camera_ids=[0, 0])  # a pinhole camera of a mixed file
    empty = CM.undistort_frames(torch.zeros(0, 6, 8, 3, dtype=torch.uint8), u)  # nothing to do: no device needed
    assert empty.shape == (0, 6, 8, 3) and empty.dtype == torch.uint8
    with pytest.raises(ValueError):
        CM.Undistortion(8, 6, _K(10, 10, 4, 3), [0.1] * 5, 1)
    with pytest.raises(ValueError):
        CM.Undistortion(8, 6, _K(10, 10, 4, 3), [0.1] * 4, 2)


def test_abi_argument_errors_without_a_gpu():
    from gssdf_b200 import _lib
    L = _lib.lib()
    assert L.gssdf_abi_revision() == 18
    dummy = 1 << 20  # never dereferenced: every call below is refused before any launch

    def mk(**kw):
        base = dict(model=0, W=8, H=6, K=[10, 0, 4, 0, 10, 3, 0, 0, 1], D=[0.1, 0, 0, 0, 0], new_K=[10, 0, 4, 0, 10, 3, 0, 0, 1], map=dummy)
        base.update(kw)
        return _lib.make_args("gssdf_undistort_map_args", **base)

    for kw in (dict(model=2), dict(model=-1), dict(W=0), dict(H=0), dict(W=1 << 15, H=1 << 15), dict(map=None), dict(map=dummy + 2),
               dict(K=[float("nan")] + [0] * 8), dict(D=[float("inf"), 0, 0, 0, 0]), dict(new_K=[0] * 8 + [float("inf")])):
        assert L.gssdf_undistort_map(ctypes.byref(mk(**kw)), None) == -1, kw
    assert L.gssdf_undistort_map(None, None) == -1

    C = ctypes
    off = (C.c_int64 * 2)(0, 144)
    sz = (C.c_int32 * 4)(8, 6, 8, 6)
    ids = (C.c_int32 * 2)(0, 0)
    mp = (C.c_void_p * 1)(dummy)
    msz = (C.c_int32 * 2)(8, 6)

    def mk8(**kw):
        base = dict(n_frames=2, n_bytes=288, src=dummy, dst=dummy + 4096, offsets=C.addressof(off), sizes=C.addressof(sz),
                    map_ids=C.addressof(ids), n_maps=1, maps=C.addressof(mp), map_sizes=C.addressof(msz))
        base.update(kw)
        return _lib.make_args("gssdf_undistort_u8_args", **base)

    bad_off = (C.c_int64 * 2)(0, 145)
    neg_off = (C.c_int64 * 2)(-3, 144)
    bad_ids = (C.c_int32 * 2)(0, 1)
    bad_sz = (C.c_int32 * 4)(8, 6, 0, 6)
    bad_msz = (C.c_int32 * 2)(8, 5)
    bad_mp = (C.c_void_p * 1)(dummy + 4)
    for kw in (dict(n_frames=-1), dict(src=None), dict(dst=None), dict(offsets=None), dict(sizes=None), dict(map_ids=None),
               dict(maps=None), dict(map_sizes=None), dict(n_maps=0), dict(n_bytes=287), dict(dst=dummy + 100),
               dict(offsets=C.addressof(bad_off)), dict(offsets=C.addressof(neg_off)), dict(map_ids=C.addressof(bad_ids)),
               dict(sizes=C.addressof(bad_sz)), dict(map_sizes=C.addressof(bad_msz)), dict(maps=C.addressof(bad_mp))):
        assert L.gssdf_undistort_u8(ctypes.byref(mk8(**kw)), None) == -1, kw
    assert L.gssdf_undistort_u8(ctypes.byref(mk8(n_frames=0, src=None)), None) == 0  # an empty batch is a no-op
    assert L.gssdf_undistort_u8(None, None) == -1
