"""The render background and the image mask on the GPU (DESIGN 7o): the post-op's composite against ATen's evaluation of NeuralGS::render's
expressions (neural_gaussian.cpp:545-553) bit for bit, its backward against torch autograd, the masked L1 and DSSIM terms against fp64
restatements of loss.cpp:22-47, GsTrainer end to end on an open-top box room (white sky) and with a corrupted, masked-out image region,
the random background's redraw and replay, and where the iterations synchronise with both options on."""
import math

import numpy as np
import pytest
import torch

from gssdf_b200 import cabi
from gssdf_b200 import gs_init as GI
from gssdf_b200 import gstrain as GT
from gssdf_b200 import metrics as MT
from gssdf_b200 import nsdf as NS
from gssdf_b200 import octree as OT
from gssdf_b200 import scene as S
from gssdf_b200 import sdf as SD
from render_shapes import window_1d

pytestmark = pytest.mark.gpu
f32 = np.float32
LEAF, BCE_SIGMA = 0.05, 0.01
W, H = 160, 120


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


# ---- kernels -------------------------------------------------------------------------------------------------------------------------
def _post_inputs(C, Hh, Ww, seed):
    dev = _dev()
    g = torch.Generator(dev).manual_seed(seed)
    r = lambda *s: torch.rand(*s, device=dev, generator=g)
    alphas = 0.2 + 0.8 * r(C, Hh, Ww, 1)
    vm = torch.eye(4, device=dev).repeat(C, 1, 1)
    vm[:, :3, :3] = torch.linalg.qr(torch.randn(C, 3, 3, device=dev, generator=g))[0]
    return dict(viewmats=vm.contiguous(), colors=r(C, Hh, Ww, 3), depths=3 * r(C, Hh, Ww, 1) * alphas, alphas=alphas,
                normals=r(C, Hh, Ww, 3) - 0.5, bg=r(C, Hh, Ww, 3))


def _post_fwd(x, mode, plain=False):
    C, Hh, Ww = x["colors"].shape[:3]
    out, nrm = torch.empty(C, Hh, Ww, 4, device=x["colors"].device), torch.empty(C, Hh, Ww, 3, device=x["colors"].device)
    args = (C, Ww, Hh, x["viewmats"], x["colors"], x["depths"], x["alphas"], x["normals"], out, nrm)
    if plain:
        cabi.render_post_fwd(*args)
    else:
        cabi.render_post_bg_fwd(*args, mode, x["bg"] if mode == 2 else None)
    return out, nrm


def test_background_forward_is_atens_composition():
    """Modes 1 and 2 give the bits of c + (1 - a) and c + (1 - a) * bg evaluated by ATen on the same device tensors; expected depth and
    normals are those of the plain post-op; mode 0 through the new entry point is the plain post-op."""
    x = _post_inputs(2, 37, 53, 1)
    base, base_n = _post_fwd(x, 0, plain=True)
    for mode in (0, 1, 2):
        out, nrm = _post_fwd(x, mode)
        c, a = x["colors"], x["alphas"]
        ref = c if mode == 0 else (c + (1.0 - a) if mode == 1 else c + (1.0 - a) * x["bg"])
        assert torch.equal(out[..., :3], ref), mode
        assert torch.equal(out[..., 3], base[..., 3]) and torch.equal(nrm, base_n), mode
    assert torch.equal(_post_fwd(x, 0)[0], base)


@pytest.mark.parametrize("mode", [1, 2])
def test_background_backward_matches_autograd(mode):
    """v_render_alphas and v_render_colors of the background post backward against torch autograd (fp32, same device) of the composite
    followed by the plain post-op's expected depth, with a direct alpha cotangent as well. Bound: 8 fp32 ulps of the cotangent's largest
    entry (the kernel and autograd sum the alpha terms in different orders)."""
    dev = _dev()
    C, Hh, Ww = 2, 37, 53
    x = _post_inputs(C, Hh, Ww, 2 + mode)
    g = torch.Generator(dev).manual_seed(9)
    v_out = torch.randn(C, Hh, Ww, 4, device=dev, generator=g)
    v_nrm = torch.randn(C, Hh, Ww, 3, device=dev, generator=g)
    v_a_in = torch.randn(C, Hh, Ww, 1, device=dev, generator=g)
    outs = dict(c=torch.empty(C, Hh, Ww, 3, device=dev), d=torch.empty(C, Hh, Ww, 1, device=dev), a=torch.empty(C, Hh, Ww, 1, device=dev),
                n=torch.empty(C, Hh, Ww, 3, device=dev))
    cabi.render_post_bg_bwd(C, Ww, Hh, x["viewmats"], x["depths"], x["alphas"], v_out, v_nrm, v_a_in, outs["c"], outs["d"], outs["a"],
                            outs["n"], mode, x["bg"] if mode == 2 else None)
    plain = {k: torch.empty_like(v) for k, v in outs.items()}
    cabi.render_post_bwd(C, Ww, Hh, x["viewmats"], x["depths"], x["alphas"], v_out, v_nrm, v_a_in, plain["c"], plain["d"], plain["a"],
                         plain["n"])
    c = x["colors"].clone().requires_grad_(True)
    a = x["alphas"].clone().requires_grad_(True)
    d = x["depths"].clone().requires_grad_(True)
    rgb = c + (1.0 - a) if mode == 1 else c + (1.0 - a) * x["bg"]
    ed = (d / a).nan_to_num()
    ((rgb * v_out[..., :3]).sum() + (ed * v_out[..., 3:]).sum() + (a * v_a_in).sum()).backward()
    assert torch.equal(outs["c"], v_out[..., :3]) and torch.equal(outs["c"], c.grad)
    bound = 8 * 2.0 ** -23 * float(a.grad.abs().max())
    err = float((outs["a"] - a.grad).abs().max())
    assert err <= bound, (err, bound)
    assert torch.equal(outs["d"], plain["d"]) and torch.equal(outs["n"], plain["n"])
    # the background's term is what the plain backward lacks
    bgv = v_out[..., :3] if mode == 1 else v_out[..., :3] * x["bg"]
    assert float((outs["a"] - (plain["a"] - bgv.sum(-1, keepdim=True))).abs().max()) <= bound


def _sep_conv(t, w):
    """depthwise conv2d of t [B, 3, H, W] with the window outer(w, w), zero padding 5, as 11 + 11 shifted adds (autograd-friendly)."""
    Hh, Ww = t.shape[-2:]
    p = torch.nn.functional.pad(t, (5, 5, 0, 0))
    h = sum(float(w[k]) * p[..., :, k:k + Ww] for k in range(11))
    p = torch.nn.functional.pad(h, (0, 0, 5, 5))
    return sum(float(w[k]) * p[..., k:k + Hh, :] for k in range(11))


def _dssim_ref_masked(x, y, w_dssim, mask):
    """test_gpu_loss_shapes._dssim_ref with loss.cpp:40-43's mask: 1 - ssim(pred * m, gt * m) in fp64; mask [H,W,3] bool."""
    w = window_1d()
    m = mask.double().permute(2, 0, 1)[None]
    xr = x[..., :3].double().permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    xm = xr * m
    yr = y[..., :3].double().permute(0, 3, 1, 2).contiguous() * m
    mu1, mu2 = _sep_conv(xm, w), _sep_conv(yr, w)
    s1 = _sep_conv(xm * xm, w) - mu1 * mu1
    s2 = _sep_conv(yr * yr, w) - mu2 * mu2
    s12 = _sep_conv(xm * yr, w) - mu1 * mu2
    ssim = ((2 * mu1 * mu2 + 1e-4) * (2 * s12 + 9e-4)) / ((mu1 * mu1 + mu2 * mu2 + 1e-4) * (s1 + s2 + 9e-4))
    ref = w_dssim * (1 - ssim.mean())
    ref.backward()
    return float(ref), xr.grad


def _loss_inputs(C, Hh, Ww, seed):
    dev = _dev()
    g = torch.Generator(dev).manual_seed(seed)
    x = torch.rand(C, Hh, Ww, 4, device=dev, generator=g)
    y = (x + 0.2 * torch.randn(C, Hh, Ww, 4, device=dev, generator=g)).clamp(0, 1).contiguous()
    mask = torch.rand(Hh, Ww, 1, device=dev, generator=g).gt(0.2).expand(Hh, Ww, 3).contiguous()
    mask[Hh // 4:Hh // 2, Ww // 3:Ww // 2] = False
    mask[3, 7, 1] = False
    return x, y, mask


def _losses(x, y, mask, w_rgb=0.8, w_depth=0.1, w_dssim=0.2):
    """masked (mask given) or plain L1 + DSSIM, as SplatRenderer.backward runs them: (loss, colour cotangent)"""
    C, Hh, Ww = x.shape[:3]
    loss, v = torch.zeros(1, device=x.device), torch.empty_like(x)
    ws = cabi.Workspace(x.device)
    if mask is None:
        cabi.l1_loss(C, Ww, Hh, x, y, w_rgb, w_depth, loss, v)
        cabi.dssim_loss(C, Ww, Hh, x, y, w_dssim, loss, v, ws)
    else:
        m8 = mask.to(torch.uint8).contiguous()
        cabi.l1_loss_masked(C, Ww, Hh, x, y, w_rgb, w_depth, loss, v, m8)
        cabi.dssim_loss_masked(C, Ww, Hh, x, y, w_dssim, loss, v, ws, m8)
    return loss, v


@pytest.mark.parametrize("W_,H_,C", [(160, 120, 1), (1200, 680, 1), (301, 77, 2)])
def test_masked_losses_against_fp64(W_, H_, C):
    """Loss and colour cotangent of the masked L1 + DSSIM against an fp64 composition of loss.cpp's masked expressions (the loss to 1e-5
    relative, the cotangent to 1e-4 of its largest entry: test_gpu_loss_shapes' DSSIM bounds); the cotangent is exactly 0 where the mask
    is 0 and the depth channel is the unmasked L1's."""
    x, y, mask = _loss_inputs(C, H_, W_, W_ + H_ + C)
    w_rgb, w_depth, w_dssim = 0.8, 0.1, 0.2
    loss, v = _losses(x, y, mask, w_rgb, w_depth, w_dssim)
    torch.cuda.synchronize()
    n = C * H_ * W_
    m = mask.double()
    d = (x - y).double()
    l1 = w_rgb * (d[..., :3] * m).abs().sum() / (3 * n) + w_depth * d[..., 3].abs().sum() / n
    ds, grad = _dssim_ref_masked(x, y, w_dssim, mask)
    ref = float(l1) + ds
    assert abs(float(loss) - ref) <= 1e-5 * abs(ref), (float(loss), ref)
    g_ref = (w_rgb / (3 * n)) * torch.sign(d[..., :3] * m) * m + grad.permute(0, 2, 3, 1)
    err = float((v[..., :3].double() - g_ref).abs().max())
    assert err <= 1e-4 * float(g_ref.abs().max()), err
    assert (v[..., :3][~mask.expand(C, -1, -1, -1)] == 0).all()
    sd = float(f32(f32(w_depth) / f32(n)))  # the kernel's fp32 scale
    assert torch.equal(v[..., 3], sd * torch.sign(x[..., 3] - y[..., 3]))


def test_all_ones_mask_is_the_unmasked_loss():
    """An all-ones mask gives the unmasked entry points' bits: the cotangents at training sizes, and the losses where their reductions
    have one order (one L1 CTA, one DSSIM warp per channel; at larger sizes the float atomics' order varies from run to run)."""
    x, y, _ = _loss_inputs(2, 120, 160, 5)
    for C, Hh, Ww in ((2, 120, 160), (1, 8, 16)):
        xs, ys = x[:C, :Hh, :Ww].contiguous(), y[:C, :Hh, :Ww].contiguous()
        ones = torch.ones(Hh, Ww, 3, dtype=torch.bool, device=x.device)
        la, va = _losses(xs, ys, None)
        lb, vb = _losses(xs, ys, ones)
        torch.cuda.synchronize()
        assert torch.equal(va, vb), (C, Hh, Ww)
        if Hh * Ww <= 256:
            assert torch.equal(la, lb)
        else:
            assert abs(float(la) - float(lb)) <= 1e-6 * abs(float(la))


# ---- the trainer ---------------------------------------------------------------------------------------------------------------------
def _poses(n, seed):
    """Cameras anywhere in the inner half of the box room, any yaw, pitch within +-0.5 rad (OpenCV axes), c2w [n,4,4] float32."""
    rng = np.random.default_rng(seed)
    c2w = np.zeros((n, 4, 4), np.float32)
    for i in range(n):
        yaw, pitch = rng.uniform(0, 2 * math.pi), rng.uniform(-0.5, 0.5)
        f = np.array([math.cos(pitch) * math.cos(yaw), math.cos(pitch) * math.sin(yaw), math.sin(pitch)])
        right = np.cross(f, [0.0, 0.0, 1.0])
        right /= np.linalg.norm(right)
        c2w[i, :3, :3] = np.stack([right, np.cross(f, right), f], 1)
        c2w[i, :3, 3] = rng.uniform(-0.5, 0.5, 3) * S.BOX
        c2w[i, 3, 3] = 1.0
    return torch.from_numpy(c2w)


def _K():
    return torch.tensor([[W / 2.0, 0, (W - 1) / 2.0], [0, W / 2.0, (H - 1) / 2.0], [0, 0, 1.0]], dtype=torch.float32)


def _images(c2w):
    return S.box_room_color(c2w.to(_dev()), W / 2.0, W / 2.0, (W - 1) / 2.0, (H - 1) / 2.0, W, H)


def _sky(c2w):
    """[B,H,W] bool: the pixels whose ray leaves the box room through its ceiling (z = +BOX[2])."""
    dev = _dev()
    j = torch.arange(W, dtype=torch.float64, device=dev)
    i = torch.arange(H, dtype=torch.float64, device=dev)
    dc = torch.stack([((j[None, :] - (W - 1) / 2.0) / (W / 2.0)).expand(H, W), ((i[:, None] - (H - 1) / 2.0) / (W / 2.0)).expand(H, W),
                      torch.ones(H, W, dtype=torch.float64, device=dev)], -1)
    P = c2w.to(dev, torch.float64)
    o, d = P[:, None, None, :3, 3], torch.einsum("brc,hwc->bhwr", P[:, :3, :3], dc)
    box = torch.as_tensor(S.BOX, dtype=torch.float64, device=dev)
    t = torch.where(d > 0, (box - o) / d, torch.where(d < 0, (-box - o) / d, torch.full_like(d, float("inf"))))
    return (t.argmin(-1) == 2) & (d[..., 2] > 0)


def _open_top_images(c2w):
    """The box room without its ceiling: the sky is white (1.0), everything else box_room_color."""
    imgs = _images(c2w)
    imgs[_sky(c2w)] = 1.0
    return imgs


def _room(open_top):
    dev = _dev()
    pack = S.box_room_pack(dev, 120, ds_pt_num=2000, seed=0)
    if open_top:  # no depth returns from the sky: no points, no octree leaves and no splats up there
        keep = pack["xyz"][:, 2] < float(S.BOX[2]) - 1e-3
        pack = {k: v[keep].contiguous() for k, v in pack.items()}
    tree, frame, _ = OT.build_occ_map(pack["xyz"], pack["depth"], 0.01, 100.0, 14.0, LEAF)
    pos = np.asarray(frame["origin"], f32)
    lo = tuple(float(f32(pos[k] + f32(frame["xyz_min_M"][k]))) for k in range(3))
    hi = tuple(float(f32(pos[k] + f32(frame["xyz_max_M"][k]))) for k in range(3))
    margin = (tuple(float(f32(f32(v) + f32(0.5 * LEAF))) for v in frame["xyz_min_M"]),
              tuple(float(f32(f32(v) - f32(0.5 * LEAF))) for v in frame["xyz_max_M"]))
    return dict(pack=pack, tree=tree, frame=frame, lo=lo, hi=hi, margin=margin)


@pytest.fixture(scope="module")
def room():
    return _room(False)


@pytest.fixture(scope="module")
def open_room():
    return _room(True)


def _sdf_trainer(room, iters, seed=0, **kw):
    fr = room["frame"]
    net = SD.SdfNet(_dev(), origin=fr["origin"], map_size=fr["map_size"], bce_isigma=1.0 / BCE_SIGMA, seed=1337 + seed)
    T = NS.SdfTrainer(net, room["tree"], room["pack"], iters, leaf_size=LEAF, bce_sigma=BCE_SIGMA, xyz_min=room["lo"], xyz_max=room["hi"],
                      seed=seed, **kw)
    T.run()
    return T


def _splats(room, S_, sh_degree, vis_batch_pt_num=20000):
    fr = room["frame"]
    net = S_.write_back()
    sp, _ = GI.neural_gs_init(room["tree"], net, room["margin"], LEAF, vis_batch_pt_num=vis_batch_pt_num, sh_degree=sh_degree,
                              spatial_scale=0.5 * fr["inner_map_size"], inner_map_size=fr["inner_map_size"], map_origin=fr["origin"], sky=False,
                              generator=torch.Generator(_dev()).manual_seed(0))
    return sp


def _gs_trainer(room, S_, frames, iters, sh_degree=1, capacity_mult=3, **kw):
    sp = _splats(room, S_, sh_degree)
    c2w, imgs = frames
    fr = room["frame"]
    return GT.GsTrainer(S_, sp, c2w, _K(), imgs, capacity=capacity_mult * sp["anchors"].shape[0], spatial_scale=0.5 * fr["inner_map_size"],
                        gs_iter_step=iters, sh_degree=sh_degree, **kw)


SHRUNK = dict(refine_gs_struct_start_iter=3, sh_degree_interval=5, outlier_remove=True, outlier_removal_interval=10,
              densify=dict(refine_start_iter=2, refine_every=4, reset_alpha_every=2, pause_refine_after_reset=0, grow_grad2d=1e-6))
E2E = dict(sh_degree=1, capacity_mult=32, outlier_remove=True, refine_gs_struct_start_iter=500, sh_degree_interval=250,
           densify=dict(refine_start_iter=100, refine_every=100))


def _held_out_psnr(G, c2w, imgs):
    st = G.state()
    vms = torch.linalg.inv(c2w.to(torch.float64)).to(torch.float32)
    renders = torch.stack([st["render"](vm) for vm in vms])
    full, _ = MT.eval_render(renders.clamp(0, 1), imgs, [f"{i}.png" for i in range(len(vms))])
    return full["PSNR"]


def test_white_background_end_to_end_on_an_open_top_room(open_room):
    """SdfTrainer (200 iterations) on the box room without its ceiling -> neural_gs_init -> GsTrainer (colour init + 1000 joint
    iterations, 40 training views at 160x120) twice from the same SDF stage, with bck_color 1 and 0; PSNR over 10 held-out views whose
    sky is white. Mode 0 composites the transparent sky black against a white ground truth. Measured on an H100 80GB HBM3 (700 W): mode 1
    32.6 dB, mode 0 26.1 dB; the bounds are 28 dB and a 4 dB margin."""
    c2w = _poses(50, 21)
    imgs = _open_top_images(c2w)
    assert 0.03 < float(_sky(c2w).float().mean()) < 0.5  # the held-out and training views see sky
    train, test = slice(0, 40), slice(40, 50)
    psnr = {}
    for mode in (1, 0):
        S_ = _sdf_trainer(open_room, 200, seed=5, outlier_remove=True)
        G = _gs_trainer(open_room, S_, (c2w[train].contiguous(), imgs[train].contiguous()), 1000, bck_color=mode, **E2E)
        G.run()
        assert np.isfinite(G.histories()["loss"]).all()
        psnr[mode] = _held_out_psnr(G, c2w[test], imgs[test])
    print(f"held-out PSNR: bck_color 1 {psnr[1]:.2f} dB, bck_color 0 {psnr[0]:.2f} dB")
    assert psnr[1] > 28.0 and psnr[1] > psnr[0] + 4.0


def test_masked_corruption_end_to_end(room):
    """A fixed rectangle of every training image (a quarter of the frame) replaced by noise: GsTrainer (1000 joint iterations, 40 views)
    with a mask that excludes it scores on clean held-out views close to a run on the clean images, and clearly above an unmasked run on
    the corrupted ones. Measured on an H100 80GB HBM3 (700 W): clean 32.4 dB, masked 29.1 dB, unmasked 25.0 dB (the masked run sees
    three quarters of the pixels per iteration, so it converges more slowly); the bounds are masked >= clean - 4.5 dB and masked >=
    unmasked + 2.5 dB."""
    dev = _dev()
    c2w = _poses(50, 23)
    imgs = _images(c2w)
    train, test = slice(0, 40), slice(40, 50)
    r0, r1, c0, c1 = H // 4, 3 * H // 4, W // 4, 3 * W // 4
    bad = imgs[train].clone()
    bad[:, r0:r1, c0:c1] = torch.rand(bad[:, r0:r1, c0:c1].shape, device=dev, generator=torch.Generator(dev).manual_seed(1))
    mask = torch.ones(H, W, dtype=torch.bool, device=dev)
    mask[r0:r1, c0:c1] = False
    psnr = {}
    for name, frames, m in (("clean", imgs[train], None), ("masked", bad, mask), ("unmasked", bad, None)):
        S_ = _sdf_trainer(room, 200, seed=5, outlier_remove=True)
        G = _gs_trainer(room, S_, (c2w[train].contiguous(), frames.contiguous()), 1000, mask=m, **E2E)
        G.run()
        assert np.isfinite(G.histories()["loss"]).all()
        psnr[name] = _held_out_psnr(G, c2w[test], imgs[test])
    print("held-out PSNR: " + ", ".join(f"{k} {v:.2f} dB" for k, v in psnr.items()))
    assert psnr["masked"] > psnr["clean"] - 4.5 and psnr["masked"] > psnr["unmasked"] + 2.5


def test_random_background_redraws_and_replays(room):
    """bck_color 2: consecutive renders composite different backgrounds, re-seeding `bg_gen` replays a render bit for bit, the splat
    samples' stream is that of mode 0, and a short run (colour initialisation and 12 joint iterations) ends with finite losses."""
    S_ = _sdf_trainer(room, 200, seed=5)
    c2w = _poses(6, 25)
    G = _gs_trainer(room, S_, (c2w, _images(c2w)), 12, bck_color=2, **SHRUNK)
    G.run()
    h = G.histories()
    assert np.isfinite(h["loss"]).all() and np.isfinite(h["color_loss"]).all() and np.isfinite(h["sdf_loss"]).all()
    vm = torch.linalg.inv(c2w[0].to(torch.float64)).to(torch.float32)
    a, bg_a = G.render(vm), G.T.bg.clone()
    b, bg_b = G.render(vm), G.T.bg.clone()
    assert not torch.equal(bg_a, bg_b) and not torch.equal(a, b)
    assert float(bg_a.min()) >= 0.0 and float(bg_a.max()) < 1.0 and abs(float(bg_a.mean()) - 0.5) < 0.01
    G.bg_gen.manual_seed(77)
    c = G.render(vm)
    G.bg_gen.manual_seed(77)
    assert torch.equal(G.render(vm), c)
    # the background draws come from their own generator: the randns stream is the seed's, as in modes 0 and 1
    ref = torch.Generator(_dev()).manual_seed(0)
    r = torch.empty_like(G.randns)
    for _ in range(12):
        r.normal_(generator=ref)
    assert torch.equal(r, G.randns)


@pytest.mark.parametrize("bck_color", [1, 2])
def test_iterations_synchronise_only_where_the_reference_reads_back(room, bck_color):
    """test_gpu_gs_train's synchronisation check with a background and an image mask: under torch.cuda.set_sync_debug_mode("error") the
    iterations of a 40-iteration run synchronise only inside the NaN prune's read, a due invisible prune, the refinement surgery and the
    outlier removal (each allowed while it runs)."""
    S_ = _sdf_trainer(room, 100, seed=2, outlier_remove=True)
    c2w = _poses(6, 6)
    mask = torch.ones(H, W, 1, dtype=torch.uint8, device=_dev())
    mask[:20, :30] = 0
    G = _gs_trainer(room, S_, (c2w, _images(c2w)), 40, capacity_mult=8, bck_color=bck_color, mask=mask,
                    **dict(SHRUNK, outlier_removal_interval=12))
    D = G.D

    def allowed(fn, due=lambda *a: True):
        def wrapped(*a, **kw):
            if not due(*a):
                return fn(*a, **kw)
            torch.cuda.set_sync_debug_mode("default")
            try:
                return fn(*a, **kw)
            finally:
                torch.cuda.set_sync_debug_mode("error")
        return wrapped
    D.prune_nan_gs = allowed(D.prune_nan_gs)
    D.prune_invisible_gs = allowed(D.prune_invisible_gs, lambda it: it > 0 and it % D.num_train_data == 0)
    D.grow_gs, D.prune_gs = allowed(D.grow_gs), allowed(D.prune_gs)
    S_.remove_outliers = allowed(S_.remove_outliers)
    G.run_color_init()
    G.start_rates()
    G.step(0)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for i in range(1, 40):
            G.step(i)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    h = G.histories()
    assert np.isfinite(h["loss"]).all() and (h["n_samples"] > 0).all()
    assert [e[0] for e in h["densify_events"]][:2] == [4, 8]
    assert G.T.mask.shape == (H, W, 3) and G.T.mask.dtype == torch.uint8
