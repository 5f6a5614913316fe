"""No-GPU checks of the render background and the image mask (DESIGN 7o): the four entry points are declared, exported and argument-
checked, the ABI revision is unchanged, GsTrainer and GsSdfStep reject bad options before any device work, fp64 restatements of the
composite, its alpha cotangent and the masked L1 and DSSIM terms agree with torch autograd of the reference's expressions
(neural_gaussian.cpp:545-553, loss.cpp:22-47), and the kernels the change templated compile to the parent's SASS."""
import ctypes
import os
import shutil
import subprocess
import sys
import types

import numpy as np
import pytest

torch = pytest.importorskip("torch")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

NEW = ("gssdf_render_post_bg_fwd", "gssdf_render_post_bg_bwd", "gssdf_l1_loss_masked", "gssdf_dssim_loss_masked")


def test_entry_points_are_declared_exported_and_abi_unchanged():
    from gssdf_b200 import _lib
    L = _lib.lib()
    for name in NEW:
        assert name in _lib.FUNCS and hasattr(L, name), name
    assert L.gssdf_abi_revision() == 18
    # each new struct extends the plain one by value, as its first member
    for new, base in (("gssdf_render_post_bg_fwd_args", "gssdf_render_post_fwd_args"), ("gssdf_render_post_bg_bwd_args", "gssdf_render_post_bwd_args"),
                      ("gssdf_l1_loss_masked_args", "gssdf_l1_loss_args"), ("gssdf_dssim_loss_masked_args", "gssdf_dssim_loss_args")):
        f0 = _lib.STRUCTS[new]._fields_[0]
        assert f0[1] is _lib.STRUCTS[base] and getattr(_lib.STRUCTS[new], f0[0]).offset == 0


def test_argument_errors_without_gpu():
    from gssdf_b200 import _lib
    L = _lib.lib()
    fake = 0x1000  # never dereferenced: every check runs before the launch
    post = _lib.make_args("gssdf_render_post_fwd_args", C=1, image_width=8, image_height=8, viewmats=fake, render_colors=fake,
                          render_depths=fake, render_alphas=fake, render_normals=fake, out_colors=fake, out_normals=fake)
    for mode, bg, msg in ((3, None, b"bck_mode 3"), (-1, None, b"bck_mode -1"), (2, None, b"needs a background")):
        a = _lib.make_args("gssdf_render_post_bg_fwd_args", post=post, bck_mode=mode, bg=bg)
        assert L.gssdf_render_post_bg_fwd(ctypes.byref(a), None) == -1
        assert msg in L.gssdf_last_error()
    bpost = _lib.make_args("gssdf_render_post_bwd_args", C=1, image_width=8, image_height=8, viewmats=fake, render_depths=fake,
                           render_alphas=fake, v_out_colors=fake, v_out_normals=fake, v_render_colors=fake, v_render_depths=fake,
                           v_render_alphas=fake, v_render_normals=fake)
    a = _lib.make_args("gssdf_render_post_bg_bwd_args", post=bpost, bck_mode=2)
    assert L.gssdf_render_post_bg_bwd(ctypes.byref(a), None) == -1 and b"needs a background" in L.gssdf_last_error()
    assert L.gssdf_render_post_bg_fwd(None, None) == -1 and L.gssdf_render_post_bg_bwd(None, None) == -1
    # the plain call's checks apply through the nested struct
    a = _lib.make_args("gssdf_render_post_bg_fwd_args", post=_lib.make_args("gssdf_render_post_fwd_args", C=0), bck_mode=1)
    assert L.gssdf_render_post_bg_fwd(ctypes.byref(a), None) == -1 and b"bad image size" in L.gssdf_last_error()
    l1 = _lib.make_args("gssdf_l1_loss_args", C=1, image_width=8, image_height=8, out_colors=fake, gt=fake, loss_out=fake, v_out_colors=fake)
    a = _lib.make_args("gssdf_l1_loss_masked_args", loss=l1, mask=None)
    assert L.gssdf_l1_loss_masked(ctypes.byref(a), None) == -1 and b"null mask" in L.gssdf_last_error()
    ds = _lib.make_args("gssdf_dssim_loss_args", C=1, image_width=8, image_height=8, out_colors=fake, gt=fake, loss_out=fake)
    a = _lib.make_args("gssdf_dssim_loss_masked_args", loss=ds, mask=None)
    assert L.gssdf_dssim_loss_masked(ctypes.byref(a), None) == -1 and b"null mask" in L.gssdf_last_error()
    a = _lib.make_args("gssdf_dssim_loss_masked_args", loss=_lib.make_args("gssdf_dssim_loss_args", C=1, image_width=8, image_height=8),
                       mask=fake)
    assert L.gssdf_dssim_loss_masked(ctypes.byref(a), None) == -1 and b"null pointer" in L.gssdf_last_error()


def _bad_options(H, W):
    """(kwargs, message) pairs every entry point must refuse; CPU tensors only."""
    cuda = torch.device("cuda:0")
    return [
        (dict(bck_color=3), "bck_color"), (dict(bck_color=-1), "bck_color"), (dict(bck_color=True), "bck_color"),
        (dict(bck_color="white"), "bck_color"),
        (dict(mask=torch.ones(H, W)), "bool or uint8"), (dict(mask=np.ones((H, W), bool)), "bool or uint8"),
        (dict(mask=torch.ones(H, W, 2, dtype=torch.bool)), r"\[H,W\]"), (dict(mask=torch.ones(W, H, dtype=torch.uint8)), r"\[H,W\]"),
        (dict(mask=torch.ones(1, H, W, 3, dtype=torch.bool)), r"\[H,W\]"),
        (dict(mask=torch.ones(H, W, 3, dtype=torch.uint8)), f"on {cuda}"), (dict(mask=torch.ones(H, W, dtype=torch.bool)), "on cuda"),
    ]


def test_gs_sdf_step_rejects_bad_options():
    from gssdf_b200 import render as RD
    H, W = 12, 20
    for kw, msg in _bad_options(H, W):
        with pytest.raises(ValueError, match=msg):
            RD.GsSdfStep(100, 4, W, H, torch.device("cuda:0"), 1000, {}, **kw)


def test_gs_trainer_rejects_bad_options():
    from gssdf_b200 import gstrain as GT
    H, W = 12, 20
    sdf = types.SimpleNamespace(dev=torch.device("cuda:0"))  # nothing past the option checks is reached
    imgs = torch.zeros(2, H, W, 3)
    for kw, msg in _bad_options(H, W):
        with pytest.raises(ValueError, match=msg):
            GT.GsTrainer(sdf, {}, torch.eye(4).repeat(2, 1, 1), torch.eye(3), imgs, capacity=10, spatial_scale=1.0, **kw)


# ---- restatements ----------------------------------------------------------------------------------------------------------------------
def _composite_np(c, a, mode, bg):
    """The post-op's colour: each step one rounding in the dtype of the inputs (fp32: the kernel's __fsub_rn / __fmul_rn / __fadd_rn)."""
    one = c.dtype.type(1)
    t = one - a
    return c + t if mode == 1 else c + t * bg


def _v_alpha_np(v, mode, bg):
    return -(v.sum(-1, keepdims=True) if mode == 1 else (v * bg).sum(-1, keepdims=True))


@pytest.mark.parametrize("mode", [1, 2])
def test_composite_and_alpha_cotangent_match_autograd(mode):
    rng = np.random.default_rng(mode)
    H, W = 7, 9
    c, a = rng.random((H, W, 3)), rng.random((H, W, 1))
    bg, v = rng.random((H, W, 3)), rng.standard_normal((H, W, 3))
    ct, at = torch.tensor(c, requires_grad=True), torch.tensor(a, requires_grad=True)
    bgt = torch.tensor(bg)
    ref = ct + (1.0 - at) if mode == 1 else ct + (1.0 - at) * bgt  # neural_gaussian.cpp:547-550
    ref.backward(torch.tensor(v))
    assert np.abs(_composite_np(c, a, mode, bg) - ref.detach().numpy()).max() <= 1e-15
    assert np.abs(_v_alpha_np(v, mode, bg) - at.grad.numpy()).max() <= 1e-14
    assert np.array_equal(ct.grad.numpy(), v)  # the colour cotangent passes through
    # in fp32 the step-by-step rounding is ATen's evaluation of the same expression, bit for bit
    c32, a32, bg32 = c.astype(np.float32), a.astype(np.float32), bg.astype(np.float32)
    t32 = torch.tensor(c32) + (1.0 - torch.tensor(a32)) if mode == 1 else torch.tensor(c32) + (1.0 - torch.tensor(a32)) * torch.tensor(bg32)
    assert np.array_equal(_composite_np(c32, a32, mode, bg32), t32.numpy())


def _mask(rng, H, W):
    m = (rng.random((H, W, 1)) > 0.3).repeat(3, -1)
    m[2:5, 3:9] = False  # a rectangle, as an image mask has
    m[0, 0, 1] = False   # and one channel alone
    return m


def test_masked_l1_matches_autograd():
    rng = np.random.default_rng(3)
    C, H, W, w = 2, 11, 13, 0.8
    r, g = rng.random((C, H, W, 3)), rng.random((C, H, W, 3))
    m = _mask(rng, H, W)
    mf = m.astype(np.float64)
    loss = w * np.abs((r - g) * mf).sum() / (3 * C * H * W)
    grad = w / (3 * C * H * W) * np.sign(r - g) * mf
    rt = torch.tensor(r, requires_grad=True)
    ref = w * torch.abs((rt - torch.tensor(g)) * torch.tensor(m)).mean()  # loss.cpp:24-26 (bool mask)
    ref.backward()
    assert abs(loss - float(ref.detach())) <= 1e-15
    assert np.abs(grad - rt.grad.numpy()).max() <= 1e-18
    assert (rt.grad.numpy()[~m[None].repeat(C, 0)] == 0).all()


def test_masked_dssim_matches_autograd():
    """1 - ssim(pred * m, gt * m) with the reference's window; the restatement is the unmasked one (bench.cpu_dssim) on the masked
    images, its gradient multiplied by m."""
    import bench
    rng = np.random.default_rng(4)
    H, W, w = 30, 37, 0.2
    x = rng.random((H, W, 3))
    y = np.clip(x + 0.2 * rng.standard_normal((H, W, 3)), 0, 1)
    m = _mask(rng, H, W)
    mf = m.astype(np.float64)
    parts = [bench.cpu_dssim(x[..., k] * mf[..., k], y[..., k] * mf[..., k], w) for k in range(3)]
    loss = w - sum(w - p[0] for p in parts) / 3  # w * (1 - mean over the three channels)
    grad = np.stack([p[1].astype(np.float64) / 3 for p in parts], -1) * mf  # cpu_dssim's mean runs over one channel
    win1 = torch.tensor([np.exp(-(np.floor((i - 11) / 2.0) ** 2) / 4.5) for i in range(11)], dtype=torch.float32)
    win1 = (win1 / win1.sum()).double()
    win = (win1[:, None] @ win1[None, :])[None, None].repeat(3, 1, 1, 1)
    xt = torch.tensor(x, requires_grad=True)
    mt = torch.tensor(m)
    p_ = (xt * mt).permute(2, 0, 1)[None]
    g_ = (torch.tensor(y) * mt).permute(2, 0, 1)[None]
    conv = lambda t: torch.nn.functional.conv2d(t, win, padding=5, groups=3)
    mu1, mu2 = conv(p_), conv(g_)
    s1, s2, s12 = conv(p_ * p_) - mu1 * mu1, conv(g_ * g_) - mu2 * mu2, conv(p_ * g_) - mu1 * mu2
    ssim = ((2 * mu1 * mu2 + 1e-4) * (2 * s12 + 9e-4)) / ((mu1 * mu1 + mu2 * mu2 + 1e-4) * (s1 + s2 + 9e-4))
    ref = w * (1 - ssim.mean())  # loss.cpp:40-43
    ref.backward()
    # the tolerances of test_host_losses.py: the two windows are normalised in fp32 in different summation orders, and cpu_dssim
    # rounds its gradient to fp32
    assert abs(loss - float(ref.detach())) <= 1e-7
    assert np.abs(grad - xt.grad.numpy()).max() <= 1e-6 * float(xt.grad.abs().max())
    assert (xt.grad.numpy()[~m] == 0).all()


# ---- SASS of the templated kernels ---------------------------------------------------------------------------------------------------
def test_plain_instantiations_compile_to_the_parents_sass():
    """tools/sass_compare.py against the parent of the commit that introduced the background and mask variants; skipped without nvcc,
    cuobjdump or that commit in the git history."""
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    if not (os.path.exists(os.path.join(cuda, "bin", "nvcc")) and os.path.exists(os.path.join(cuda, "bin", "cuobjdump"))
            and shutil.which("git") and os.path.isdir(os.path.join(ROOT, ".git"))):
        pytest.skip("needs nvcc, cuobjdump and the git history")
    log = subprocess.run(["git", "-C", ROOT, "log", "--format=%H", "-S", "gssdf_render_post_bg_fwd", "--", "gs-sdf_b200/csrc/raster.cu"],
                         capture_output=True, text=True)
    revs = log.stdout.split()
    if log.returncode or not revs:
        pytest.skip("the change is not committed yet")
    if subprocess.run(["git", "-C", ROOT, "rev-parse", "--verify", "-q", revs[-1] + "~1"], capture_output=True).returncode:
        pytest.skip("the parent commit is not in this clone")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "sass_compare.py"), "--rev", revs[-1] + "~1"], capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stdout + r.stderr
