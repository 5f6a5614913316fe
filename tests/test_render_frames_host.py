"""The 8-bit frames of gssdf_render_frames_u8 (DESIGN 7p) on the host: the numpy restatement (render_frames_oracle.py) against the
reference's composition run through cv2 (utils::tensor_to_cv_mat, utils::apply_colormap_to_depth), the committed TURBO table, and
views.load_camera_spec against render_camera_spec_v1's rules."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gs-sdf_b200"))
import render_frames_oracle as O  # noqa: E402

cv2 = pytest.importorskip("cv2")


def cv_convert_to(src, dtype, alpha):
    """Mat::convertTo(dst, dtype, alpha, 0) through the bindings: cv2.normalize(NORM_MINMAX) calls convertTo with
    scale = (dmax - dmin) / (smax - smin) and shift = dmin - smin * scale; two sentinels at -/+ 2^k and a target range of -/+ alpha 2^k
    make those exactly alpha and 0."""
    x = np.asarray(src, np.float32).ravel()
    k = int(np.ceil(np.log2(max(float(np.abs(x[np.isfinite(x)]).max(initial=0.0)), 1.0)))) + 1
    s = np.float32(2.0 ** k)
    row = np.concatenate([x, [-s, s]]).astype(np.float32).reshape(1, -1)
    out = cv2.normalize(row, None, -alpha * float(s), alpha * float(s), cv2.NORM_MINMAX, dtype=dtype)
    return out.ravel()[:-2].reshape(np.shape(src))


def cv_depth_colormap_rgb(depth):
    """apply_colormap_to_depth(tensor_to_cv_mat(depth)) of one [H,W] fp32 view, RGB."""
    mm = cv_convert_to(depth, cv2.CV_16U, 1000.0)                      # convertTo(CV_16UC1, 1000)
    d32 = mm.astype(np.float32)                                        # convertTo(CV_32FC1)
    mask = d32 > 0
    near, far, _, _ = cv2.minMaxLoc(d32, mask.astype(np.uint8))       # (far - near) < 1e-6 with the defaults near = far = 0
    alpha = 1.0 / (far - near + 1e-10)                                 # (m - near) / (far - near + 1e-10): MatOp_AddEx evaluates it as
    t = O.fma32(d32, np.float32(alpha), np.float32(-near * alpha))     # m.convertTo(m, -1, alpha, -near * alpha), fp32 fma per element
    t[~mask] = 1.0                                                     # setTo(1, ~mask)
    q = cv_convert_to(t, cv2.CV_8U, 255.0)                             # convertTo(CV_8UC1, 255)
    return cv2.applyColorMap(q.astype(np.uint8), cv2.COLORMAP_TURBO)[..., ::-1]


def test_convert_to_scale_is_an_fp32_fma():
    """convertTo(CV_32F, alpha, beta) computes fma(x, (float)alpha, (float)beta) in fp32, rounded once, and not x * alpha + beta with two
    roundings; step 4 of the colour map runs through it. Sentinels -1 and 2 with the range [0, 1] give alpha = beta = 1/3 in fp64."""
    rng = np.random.default_rng(0)
    for n in (5, 17, 33 * 17, 4099):
        x = rng.uniform(-1, 2, n).astype(np.float32)
        row = np.concatenate([x, [-1.0, 2.0]]).astype(np.float32).reshape(1, -1)
        got = cv2.normalize(row, None, 0.0, 1.0, cv2.NORM_MINMAX, dtype=cv2.CV_32F).ravel()[:-2]
        a = np.float32(1.0 / 3.0)
        assert np.array_equal(got, O.fma32(x, a, a)), n
        if n > 100:
            assert not np.array_equal(got, (x * a).astype(np.float32) + a)  # the inputs tell the two apart


def test_convert_to_rounding_and_saturation():
    """convertTo to 16U / 8U rounds half to even and saturates; NaN and values beyond int32 give 0."""
    v = np.array([0.5, 1.5, 2.5, -0.5, -3.0, 65535.4, 65535.5, 70000.0, 1e12, np.inf, np.nan], np.float32)
    assert np.array_equal(cv_convert_to(np.nan_to_num(v, nan=0, posinf=0), cv2.CV_16U, 1.0),
                          np.clip(O.cv_round(np.nan_to_num(v, nan=0, posinf=0)), 0, 65535))
    assert list(O.cv_round(v)[:4]) == [0, 2, 2, 0]
    assert O.cv_round(v)[-3:].tolist() == [-2 ** 31] * 3
    assert O.depth_mm(np.array([np.nan, np.inf, 3e6, 70.0], np.float32)).tolist() == [0, 0, 0, 65535]


def test_minmaxloc_of_an_empty_mask_is_zero():
    z = np.zeros((4, 5), np.float32)
    assert cv2.minMaxLoc(z, (z > 0).astype(np.uint8))[:2] == (0.0, 0.0)


def test_turbo_table_matches_cv2():
    lut = cv2.applyColorMap(np.arange(256, dtype=np.uint8).reshape(256, 1), cv2.COLORMAP_TURBO).reshape(256, 3)
    assert np.array_equal(O.turbo_lut_rgb(), lut[:, ::-1])


def _half_depths(rng, n):
    """fp32 depths whose fl(d * 1000) is exactly k + 0.5 (the tie of the millimetre rounding)."""
    out = []
    while len(out) < n:
        k = int(rng.integers(1, 60000))
        d = np.float32((k + 0.5) / 1000.0)
        for c in (d, np.nextafter(d, np.float32(0)), np.nextafter(d, np.float32(1e9))):
            if float(np.float32(c) * np.float32(1000)) == k + 0.5:
                out.append(c)
                break
    return np.array(out, np.float32)


def _depth_cases(rng):
    H, W = 17, 33
    cases = {
        "random": rng.uniform(0.1, 12.0, (H, W)),
        "saturating": rng.uniform(60.0, 80.0, (H, W)),
        "zero_negative": np.where(rng.random((H, W)) < 0.4, 0.0, np.where(rng.random((H, W)) < 0.5, -rng.uniform(0, 5, (H, W)),
                                                                               rng.uniform(0.2, 5, (H, W)))),
        "empty": np.where(rng.random((H, W)) < 0.5, 0.0, -1.0),
        "tiny": np.full((H, W), 0.0004),  # rounds to 0 mm: no valid pixel
        "single_value": np.where(rng.random((H, W)) < 0.5, 0.0, 2.5),
        "two_values": np.where(rng.random((H, W)) < 0.5, 1.0, 2.0),
    }
    h = _half_depths(rng, H * W).reshape(H, W)
    cases["halves"] = h
    cases["halves_and_random"] = np.where(rng.random((H, W)) < 0.5, h, rng.uniform(0.01, 70, (H, W)))
    return {k: v.astype(np.float32) for k, v in cases.items()}


def test_depth_colormap_matches_cv2():
    rng = np.random.default_rng(3)
    for name, d in _depth_cases(rng).items():
        want = cv_depth_colormap_rgb(d)
        got = O.turbo_lut_rgb()[O.depth_quantised(d)]
        assert np.array_equal(got, want), name
    for H, W in ((680, 1200), (1, 1), (7, 5)):
        d = rng.uniform(0.3, 9.0, (H, W)).astype(np.float32)
        assert np.array_equal(O.turbo_lut_rgb()[O.depth_quantised(d)], cv_depth_colormap_rgb(d)), (H, W)


def test_colour_and_normal_match_torch():
    rng = np.random.default_rng(4)
    c = rng.uniform(-0.5, 1.5, (2, 17, 33, 3)).astype(np.float32)
    c.reshape(-1)[:8] = [0.0, 1.0, np.nextafter(np.float32(1), np.float32(0)), -0.0, -1e-30, 1e-30, 254.5 / 255, 2.0]
    want = (torch.from_numpy(c).clamp(0.0, 1.0) * 255).to(torch.uint8).numpy()
    assert np.array_equal(O.trunc8(c), want)
    n = rng.uniform(-1.2, 1.2, (2, 17, 33, 3)).astype(np.float32)
    want_n = ((torch.from_numpy(n) * 0.5 + 0.5).clamp(0.0, 1.0) * 255).to(torch.uint8).numpy()
    oc = np.concatenate([c, rng.uniform(0.5, 3, (2, 17, 33, 1)).astype(np.float32)], -1)
    color, depth, normal = O.render_frames(oc, n)
    assert np.array_equal(normal, want_n) and np.array_equal(color, want)
    assert depth.shape == (2, 17, 33, 3) and depth.dtype == np.uint8


# ---- load_camera_spec ------------------------------------------------------------------------------------------------------------------
def _spec(tmp_path, text):
    p = tmp_path / "spec.txt"
    p.write_bytes(text.encode())
    return str(p)


def test_camera_spec_rules(tmp_path):
    from gssdf_b200 import views
    text = ("# whole-line comment\n\n   \n640 480 500 501 320 240  # inline comment\nnot a camera line\n"
            "320 200 250.5 251 160 100 extra tokens are ignored\n  # indented comment line is not a data line\n"
            "1280.7 720 900 900 640 360\n1280 720 900 900 640 360\n")  # an int field that reads "1280" leaves ".7": skipped
    cams = views.load_camera_spec(_spec(tmp_path, text), 3)
    assert [(w, h) for w, h, _ in cams] == [(640, 480), (320, 200), (1280, 720)]
    assert cams[1][2].tolist() == [[250.5, 0.0, 160.0], [0.0, 251.0, 100.0], [0.0, 0.0, 1.0]]
    assert cams[0][2].dtype == torch.float32


def test_camera_spec_broadcast_and_errors(tmp_path):
    from gssdf_b200 import views
    one = views.load_camera_spec(_spec(tmp_path, "64 48 50 50 32 24\n"), 5)
    assert len(one) == 5 and all((w, h) == (64, 48) for w, h, _ in one)
    two = "64 48 50 50 32 24\n32 24 25 25 16 12\n"
    with pytest.raises(ValueError, match="does not match"):
        views.load_camera_spec(_spec(tmp_path, two), 3)
    assert len(views.load_camera_spec(_spec(tmp_path, two), 2)) == 2
    for bad in ("0 48 50 50 32 24\n", "64 -1 50 50 32 24\n", "64 48 0 50 32 24\n", "64 48 50 -2 32 24\n"):
        with pytest.raises(ValueError, match="Invalid camera intrinsics"):
            views.load_camera_spec(_spec(tmp_path, bad), 1)
    assert len(views.load_camera_spec(_spec(tmp_path, "64 48 50 50 -3 -4\n"), 1)) == 1  # cx, cy are not checked
    for empty in ("", "# only a comment\n\n", "a b c d e f\n"):
        with pytest.raises(ValueError, match="no valid data lines"):
            views.load_camera_spec(_spec(tmp_path, empty), 1)
    with pytest.raises(ValueError, match="empty pose sequence"):
        views.load_camera_spec(_spec(tmp_path, "64 48 50 50 32 24\n"), 0)
    with pytest.raises(ValueError, match="does not exist"):
        views.load_camera_spec(str(tmp_path / "missing.txt"), 1)


def test_world_to_camera_is_the_fp32_inverse_of_a_rigid_pose():
    from gssdf_b200 import views
    rng = np.random.default_rng(5)
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    P = np.eye(4)
    P[:3, :3], P[:3, 3] = q, rng.normal(size=3)
    vm = views.world_to_camera(torch.tensor(P, dtype=torch.float32))
    assert vm.dtype == torch.float32 and vm[3].tolist() == [0.0, 0.0, 0.0, 1.0]
    assert np.allclose(vm.numpy().astype(np.float64), np.linalg.inv(P), atol=1e-5)
