"""export_test_image's depth-to-normal frame on the GPU (gssdf_render_depth_normal_u8, DESIGN 7p) against the fp64 restatement of
depth_normal_oracle.py: every byte within 1, and a byte that differs only where the value lies within twice the fp32 composition's own
largest deviation from fp64 of a 1/255 step; both depth sources, batches of 1 and 8, degenerate stencils, one call of C views against C
calls of one view, the argument errors, render_views(depth_normal=) against the operator on the trainer's render, and the shim twin."""
import ctypes as C

import numpy as np
import pytest
import torch

from depth_normal_oracle import export_test_image, restate
from gssdf_b200 import scene as S
from gssdf_b200 import views as VW

pytestmark = pytest.mark.gpu


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _inputs(C_, W, H, seed):
    """A smooth depth surface with noise (1..5 m), alphas in [0, 1] with a transparent share, and degenerate stencils: a zero-depth patch,
    a constant-zero row, and a constant-depth column under a camera that sees it edge-on nowhere."""
    rng = np.random.default_rng(seed)
    ys, xs = np.meshgrid(np.linspace(0, 1, H), np.linspace(0, 1, W), indexing="ij")
    depth = np.empty((C_, H, W), np.float32)
    for c in range(C_):
        base = 2.0 + np.sin(3 * xs + c) * np.cos(2 * ys) + 0.5 * xs
        depth[c] = base + 0.02 * rng.standard_normal((H, W))
    alpha = rng.random((C_, H, W)).astype(np.float32)
    alpha[rng.random((C_, H, W)) < 0.1] = 0.0
    alpha[rng.random((C_, H, W)) < 0.1] = 1.0
    if H > 8 and W > 8:
        depth[:, H // 3:H // 3 + 4, W // 4:W // 4 + 5] = 0.0
        depth[0, H // 2] = 0.0
    V, K = S.cameras(list(range(C_)), W, H)
    return depth, alpha, np.ascontiguousarray(V, np.float32), np.ascontiguousarray(K, np.float32)


def _run(depth, alpha, V, K, median):
    dev = _dev()
    C_, H, W = depth.shape
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    if median:
        d = t(depth[..., None])
    else:
        d = torch.zeros(C_, H, W, 4, device=dev)
        d[..., 3] = t(depth)
        d[..., :3] = 7.0
    return VW.render_depth_normal(d, t(alpha[..., None]), t(V), t(K)).cpu().numpy()


def _check(got, depth, alpha, V, K, label):
    want, q64 = restate(depth, alpha, V, K)
    _, q32 = export_test_image(depth, alpha, V, K, torch.float32)
    spread32 = float(np.nanmax(np.abs(q32 - q64)))
    diff = got.astype(np.int32) - want.astype(np.int32)
    assert int(np.abs(diff).max()) <= 1, f"{label}: a byte off by {int(np.abs(diff).max())}"
    bad = diff != 0
    dist = np.abs(q64 - np.maximum(got, want))  # distance of the fp64 value to the step the kernel's byte crossed
    worst = float(dist[bad].max()) if bad.any() else 0.0
    print(f"{label}: {int(bad.sum())} of {bad.size} bytes differ from fp64 by 1, farthest {worst:.3e} from the step; fp32 composition's "
          f"deviation {spread32:.3e}, its differing bytes {int((export_test_image(depth, alpha, V, K, torch.float32)[0] != want).sum())}")
    assert worst <= 2 * spread32, f"{label}: a byte differs {worst:.3e} from the step, bar {2 * spread32:.3e}"


@pytest.mark.parametrize("W,H", [(1200, 680), (1920, 1080), (33, 17)])
@pytest.mark.parametrize("C_", [1, 8])
def test_kernel_matches_the_fp64_restatement(W, H, C_):
    depth, alpha, V, K = _inputs(C_, W, H, seed=W + C_)
    med = _run(depth, alpha, V, K, True)
    ed = _run(depth, alpha, V, K, False)
    assert np.array_equal(med, ed)  # the two depth sources read the same values
    _check(med, depth, alpha, V, K, f"{W}x{H} C={C_}")
    if C_ > 1:  # one call of C views equals C calls of one view
        for c in (0, C_ - 1):
            one = _run(depth[c:c + 1], alpha[c:c + 1], V[c:c + 1], K[c:c + 1], True)
            assert np.array_equal(med[c:c + 1], one)


def test_small_and_degenerate_images():
    """1x1, 2xN and 3x3 images have no interior or a single interior pixel; zero depth everywhere gives n = 0."""
    for W, H in ((1, 1), (2, 7), (7, 2), (3, 3)):
        depth, alpha, V, K = _inputs(2, W, H, seed=W * 10 + H)
        _check(_run(depth, alpha, V, K, True), depth, alpha, V, K, f"{W}x{H}")
    depth, alpha, V, K = _inputs(1, 40, 20, seed=5)
    got = _run(np.zeros_like(depth), alpha, V, K, True)
    assert (got == 127).all()


def test_argument_errors():
    from gssdf_b200._lib import lib, make_args
    dev = _dev()
    Cn, H, W = 2, 17, 33
    d = torch.ones(Cn, H, W, 1, device=dev)
    al = torch.ones(Cn, H, W, 1, device=dev)
    V, K = S.cameras([0, 1], W, H)
    vm, Ks = torch.from_numpy(np.ascontiguousarray(V, np.float32)).to(dev), torch.from_numpy(np.ascontiguousarray(K, np.float32)).to(dev)
    out = torch.empty(Cn, H, W, 3, dtype=torch.uint8, device=dev)

    def call(**kw):
        a = dict(C=Cn, W=W, H=H, viewmats=vm, Ks=Ks, depth=d, depth_stride=1, render_alphas=al, normal=out)
        a.update(kw)
        return lib().gssdf_render_depth_normal_u8(C.byref(make_args("gssdf_render_depth_normal_args", **a)), None)
    assert call() == 0
    for kw in (dict(C=-1), dict(C=65536), dict(W=0), dict(H=0), dict(depth_stride=0), dict(depth=None), dict(normal=None),
               dict(viewmats=None), dict(Ks=None), dict(render_alphas=None), dict(depth=d.data_ptr() + 2), dict(render_alphas=al.data_ptr() + 1)):
        assert call(**kw) == -1, kw
    assert call(C=0, depth=None, normal=None, viewmats=None) == 0  # no-op
    with pytest.raises(ValueError):
        VW.render_depth_normal(torch.ones(Cn, H, W, 2, device=dev), al, vm, Ks)
    with pytest.raises(ValueError):
        VW.render_depth_normal(d, al[:1], vm, Ks)
    with pytest.raises(ValueError):
        VW.render_depth_normal(d.double(), al, vm, Ks)
    with pytest.raises(ValueError):
        VW.render_depth_normal(d, al, vm, Ks, out=out[:1])


def test_the_shim_twin_writes_the_same_bytes():
    dev = _dev()
    import gssdf_shim as shim
    depth, alpha, V, K = _inputs(3, 97, 61, seed=11)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    oc = torch.zeros(3, 61, 97, 4, device=dev)
    oc[..., 3] = t(depth)
    for d in (t(depth[..., None]), oc):
        a = VW.render_depth_normal(d, t(alpha[..., None]), t(V), t(K))
        b = shim.gssdf_render_depth_normal_frames(d, t(alpha[..., None]), t(V), t(K))
        assert torch.equal(a, b)
        one = shim.gssdf_render_depth_normal_frames(d[1], t(alpha[1, ..., None]), t(V[1]), t(K[1]))
        assert torch.equal(a[1:2], one)


# ---- after training ----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def trained():
    """A short GsTrainer run on the box room with the median-depth normal term (the helpers of test_gpu_backgrounds_masks)."""
    _dev()
    import test_gpu_backgrounds_masks as BM
    room = BM._room(False)
    c2w = BM._poses(12, seed=3)
    S_ = BM._sdf_trainer(room, 200, seed=5)
    G = BM._gs_trainer(room, S_, (c2w, BM._images(c2w)), 40, depth_type=1, refine_gs_struct_start_iter=10)
    G.run()
    return G, c2w, BM._K(), BM.W, BM.H


@pytest.mark.parametrize("depth_type", [0, 1, 3])
def test_render_views_equals_the_operator_on_the_trainers_render(trained, depth_type):
    G, c2w, K, W, H = trained
    st = G.state()
    deg = G.T.R.sh_degree
    idx = [0, 5, 11]
    got = list(VW.render_views(st["splats"], c2w[idx], (W, H, K), sh_degree=deg, depth_normal=depth_type))
    none = list(VW.render_views(st["splats"], c2w[idx], (W, H, K), sh_degree=deg))
    assert "depth2normal" not in none[0]
    R = G.T.R
    for k, i in enumerate(idx):
        vm = VW.world_to_camera(c2w[i])
        st["render"](vm)  # GsTrainer.render leaves the view's buffers in its renderer
        src = R.r["render_median"] if depth_type else R.out_colors
        want = VW.render_depth_normal(src, R.r["render_alphas"], vm[None].to(src.device), G.Ks)
        assert torch.equal(got[k]["depth2normal"], want[0].cpu()), f"view {i}"
        for name in ("color", "depth", "normal"):
            assert torch.equal(got[k][name], none[k][name])
