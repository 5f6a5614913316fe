"""Host checks of the median-depth normal term and the depth-to-normal frame (DESIGN 7o, 7p): the fp64 restatement of the frame
(tests/depth_normal_oracle.py) against an fp64 transcription of export_test_image's composition, the depth_type rule, and the argument
errors of GsTrainer and render_views that come before any device work."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")

from depth_normal_oracle import export_test_image, restate  # noqa: E402


def _camera(W, H, seed):
    """a world->camera matrix with a generic rotation and translation, and a pinhole K (fp32 values, as the kernel reads them)"""
    rng = np.random.default_rng(seed)
    q, _ = np.linalg.qr(rng.standard_normal((3, 3)))
    q *= np.sign(np.linalg.det(q))
    V = np.eye(4)
    V[:3, :3], V[:3, 3] = q, rng.standard_normal(3)
    K = np.array([[0.9 * W, 0, W / 2 + 0.3], [0, 0.9 * W, H / 2 - 0.2], [0, 0, 1]])
    return V.astype(np.float32), K.astype(np.float32)


def _agree(depth, alpha, V, K):
    got, q = restate(depth, alpha, V, K)
    want, q64 = export_test_image(depth, alpha, V, K, torch.float64)
    # the two fp64 evaluations differ in the last bits (the camera position, the matmul): bytes agree wherever the value is not within
    # 1e-9 of a truncation step
    assert float(np.abs(q - q64).max()) <= 1e-9
    near = np.abs(q64 - np.round(q64)) <= 1e-9
    assert np.array_equal(got[~near], want[~near])
    return got, q


@pytest.mark.parametrize("W,H,seed", [(33, 17, 0), (64, 48, 1), (3, 3, 2), (2, 5, 3), (1, 1, 4)])
def test_restatement_equals_the_reference_composition(W, H, seed):
    rng = np.random.default_rng(seed)
    C = 2
    V, K = zip(*[_camera(W, H, seed * 7 + c) for c in range(C)])
    V, K = np.stack(V), np.stack(K)
    depth = (1.0 + 2.0 * rng.random((C, H, W))).astype(np.float32)
    alpha = rng.random((C, H, W)).astype(np.float32)
    if H > 4 and W > 4:
        depth[0, 1:4, 1:4] = 0.0   # empty pixels: degenerate stencils
        alpha[1, 2:4, :] = 0.0     # transparent rows
    got, _ = _agree(depth, alpha, V, K)
    # border rows and columns: n = 0 -> trunc8(0.5) = 127
    assert (got[:, 0] == 127).all() and (got[:, -1] == 127).all() and (got[:, :, 0] == 127).all() and (got[:, :, -1] == 127).all()
    if H > 4 and W > 4:
        assert (got[0, 2, 2] == 127).all()  # the zero-depth stencil's normal is 0
        assert (got[1, 2:4] == 127).all()   # alpha 0


def test_truncation_at_the_steps():
    """A fronto-parallel plane seen by the identity camera has n = (0, 0, -1) exactly, so channel 2 is trunc8((1 - alpha) / 2): alphas at
    and next to the values that land on k / 255 pin the truncation (and 0.5 -> 127 in the other channels)."""
    W, H = 40, 12
    V = np.eye(4, dtype=np.float32)[None]
    K = np.array([[[30.0, 0, 20.0], [0, 30.0, 6.0], [0, 0, 1]]], np.float32)
    depth = np.full((1, H, W), 2.0, np.float32)
    ks = np.arange(0, 256, 255 / (W - 1))
    a = (1.0 - 2.0 * ks / 255.0)
    alpha = np.empty((1, H, W), np.float32)
    for r in range(H):
        alpha[0, r] = np.nextafter(a.astype(np.float32), np.float32(r % 3 - 1) * np.inf) if r % 3 != 1 else a.astype(np.float32)
    got, q = _agree(depth, alpha, V, K)
    inner = got[0, 1:-1, 1:-1]
    assert (inner[..., :2] == 127).all()
    want = np.trunc(np.clip((1.0 - alpha[0, 1:-1, 1:-1].astype(np.float64)) * 0.5, 0, 1) * 255.0)
    assert np.array_equal(inner[..., 2], want.astype(np.uint8))
    assert len(np.unique(inner[..., 2])) > 30


def test_depth_type_rule():
    from gssdf_b200.render import check_depth_type
    assert check_depth_type("t", 0) is False
    for v in (1, 3, -1, 7):
        assert check_depth_type("t", v) is True
    for bad in (0.0, 1.0, "1", None, True, False, np.float32(1)):
        with pytest.raises(ValueError, match="depth_type"):
            check_depth_type("t", bad)


def test_gs_trainer_rejects_a_bad_depth_type_before_device_work():
    from gssdf_b200 import gstrain

    class Sdf:  # only the attributes read before the depth_type check
        dev = torch.device("cuda:0")
        pack = {}
    imgs = torch.zeros(1, 4, 4, 3)
    with pytest.raises(ValueError, match="depth_type"):
        gstrain.GsTrainer(Sdf(), {}, torch.eye(4)[None], torch.eye(3), imgs, capacity=4, spatial_scale=1.0, depth_type=1.5)


def test_render_views_rejects_a_bad_depth_normal():
    from gssdf_b200 import views
    splats = dict(anchors=torch.zeros(1, 3, device="meta"))
    for bad in (1.0, "median", True):
        with pytest.raises(ValueError, match="depth_type"):
            next(views.render_views(splats, torch.eye(4)[None], (4, 4, torch.eye(3)), sh_degree=0, depth_normal=bad))
    with pytest.raises(ValueError, match="CUDA"):  # a valid selection goes on to the other checks
        next(views.render_views(splats, torch.eye(4)[None], (4, 4, torch.eye(3)), sh_degree=0, depth_normal=3))


def test_header_declares_the_entry_point():
    from gssdf_b200 import _lib
    structs, funcs, _ = _lib.parse_header()
    assert "gssdf_render_depth_normal_u8" in funcs
    fields = [f for f, _ in structs["gssdf_render_depth_normal_args"]]
    assert fields == ["C", "W", "H", "viewmats", "Ks", "depth", "depth_stride", "render_alphas", "normal"]
