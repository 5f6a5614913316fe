"""Undistortion on the GPU (DESIGN 7r): gssdf_undistort_map at every pixel of every shipped camera at full size against the numpy
restatement (undistort_oracle.py, itself equal to cv2) and against OpenCV's own map at the golden samples, and gssdf_undistort_u8 byte for
byte against the restatement: random and textured frames, cameras and sizes mixed in one batch, odd widths, W or H = 1, unaligned byte
offsets, maps that leave the frame, a pinned store staged in chunks, run-to-run identity and the libtorch twin. Then training: the box room
seen through a distorted camera trains better undistorted at the new K than distorted at the raw K."""
import os

import numpy as np
import pytest
import torch

import undistort_oracle as U
from gssdf_b200 import cabi
from gssdf_b200 import cameras as CM
from gssdf_b200 import gstrain as GT
from gssdf_b200 import metrics as MT
from gssdf_b200 import scene as S
from test_gpu_gs_train import _poses, _sdf_trainer, _splats, room  # noqa: F401  (room: the module fixture)

pytestmark = pytest.mark.gpu

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "undistort_ref.npz"))


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _K(fx, fy, cx, cy):
    return np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32)


def _shipped():
    for name, c in zip(GOLD["names"], GOLD["cams"]):
        model, W, H = int(c[0]), int(c[1]), int(c[2])
        d = np.array(c[7:12], np.float32)
        yield str(name), model, W, H, _K(*c[3:7]), d if model == 0 else d[:4]


def test_device_map_equals_the_restatement_on_every_shipped_camera():
    dev = _dev()
    for i, (name, model, W, H, K, d) in enumerate(_shipped()):
        u = CM.Undistortion(W, H, K, d, model, device=dev)
        assert np.array_equal(u.K.numpy(), GOLD["new_K"][i]), name
        got = u.map.cpu().numpy()
        ref = U.undistort_map(K, d, u.K.numpy(), model, W, H)
        bad = int((got != ref).any(-1).sum())
        assert bad == 0, f"{name}: {bad} of {W * H} map entries differ"
        flat = got.reshape(-1, 4)[GOLD["pix"][i]]
        assert np.array_equal(flat[:, :2], GOLD["map1"][i]) and np.array_equal(flat[:, 2].astype(np.uint16), GOLD["map2"][i]), name


def _texture(rng, H, W):
    y, x = np.mgrid[:H, :W]
    t = np.stack([(x * 7 + y * 3) % 256, ((x // 4 + y // 4) % 2) * 255, (np.sin(x * 0.3) * np.cos(y * 0.2) * 127 + 128)], -1)
    return t.astype(np.uint8)


def _cams(dev):
    """model-0 and model-1 cameras: an odd width, W = 1, H = 1, and zoomed-out new K whose maps leave the frame"""
    return [CM.Undistortion(61, 47, _K(52.37, 51.91, 30.83, 22.61), [-0.31, 0.11, 0.0013, -0.0021, -0.017], 0, device=dev),
            CM.Undistortion(53, 41, _K(30.11, 30.27, 26.3, 20.9), [-0.047, 0.0115, -0.0089, 0.00186], 1,
                            new_K=_K(14.9, 15.2, 26.1, 19.8), device=dev),
            CM.Undistortion(1, 37, _K(20.3, 20.1, 0.4, 18.2), [0.05, -0.01, 0.001, 0.0, 0.0], 0, device=dev),
            CM.Undistortion(29, 1, _K(15.7, 15.9, 14.1, 0.3), [0.02, 0.01, 0.003, -0.001], 1, device=dev),
            CM.Undistortion(97, 63, _K(80.2, 80.9, 47.3, 30.6), [-0.2, 0.05, 0.001, 0.002, 0.0], 0, new_K=_K(35.1, 35.3, 48.2, 31.7),
                            device=dev),
            CM.Undistortion(640, 512, _K(588.143714607, 588.107927227, 296.059369138, 254.543215481),
                            [-0.13218037625958456, 0.15360732717073536, 0.00036918417348059815, -0.00031715324469463964, 0.0], 0, device=dev)]


def _batch(rng, cams, n):
    ids = [int(i) for i in rng.integers(0, len(cams), n)]
    frames = [(rng.integers(0, 256, (cams[i].H, cams[i].W, 3), dtype=np.uint8) if k % 2 else _texture(rng, cams[i].H, cams[i].W))
              for k, i in enumerate(ids)]
    return ids, frames


def _expect(cams, ids, frames):
    return [U.remap(f, cams[i].map.cpu().numpy()) for i, f in zip(ids, frames)]


def test_remap_bytes_mixed_batch():
    dev = _dev()
    rng = np.random.default_rng(0)
    cams = _cams(dev)
    for c in cams:  # the device maps of the small cameras against the restatement too
        assert np.array_equal(c.map.cpu().numpy(), U.undistort_map(c.K_distorted, c.d, c.K.numpy(), c.model, c.W, c.H))
    ids, frames = _batch(rng, cams, 45)  # more than one launch's 32 frames
    st = GT.FramesU8.pack(frames, device=dev)
    out = CM.undistort_frames(st, cams, ids)
    assert isinstance(out, GT.FramesU8) and out.is_cuda and out.sizes == st.sizes
    for k, e in enumerate(_expect(cams, ids, frames)):
        assert np.array_equal(out.frame(k).cpu().numpy(), e), (k, ids[k])
    again = CM.undistort_frames(st, cams, ids)
    assert torch.equal(again.data, out.data)
    # the zoomed-out cameras leave the frame: their outputs hold zeros where the 2x2 block is wholly outside
    m = cams[4].map.cpu().numpy()
    assert ((m[..., 0] >= 97) | (m[..., 0] + 1 < 0) | (m[..., 1] >= 63) | (m[..., 1] + 1 < 0)).sum() > 500


def test_remap_unaligned_offsets_and_tensor_input():
    dev = _dev()
    rng = np.random.default_rng(1)
    cams = _cams(dev)
    ids, frames = _batch(rng, cams, 9)
    st = GT.FramesU8.pack(frames, device=dev)
    # shift every frame by one byte inside a larger store: offsets and the destination lose their 4-byte alignment
    n = st.data.numel()
    src = torch.zeros(n + 8, dtype=torch.uint8, device=dev)
    src[1:1 + n] = st.data
    dst = torch.full((n + 8,), 7, dtype=torch.uint8, device=dev)
    cabi.undistort_u8(src, dst, [o + 1 for o in st.offsets[:-1]], st.sizes, ids, [c.map for c in cams])
    exp = _expect(cams, ids, frames)
    for k, e in enumerate(exp):
        o = st.offsets[k] + 1
        assert np.array_equal(dst[o:o + e.size].cpu().numpy().reshape(e.shape), e), k
    assert int(dst[0]) == 7 and (dst[1 + n:] == 7).all()  # bytes outside the frames are untouched
    # a [B,H,W,3] tensor of one camera
    B = torch.from_numpy(np.stack([_texture(rng, 512, 640), rng.integers(0, 256, (512, 640, 3), dtype=np.uint8)])).to(dev)
    out = CM.undistort_frames(B, cams[5])
    assert out.shape == B.shape and out.is_cuda
    m = cams[5].map.cpu().numpy()
    for k in range(2):
        assert np.array_equal(out[k].cpu().numpy(), U.remap(B[k].cpu().numpy(), m))


def test_pinned_store_in_chunks_equals_device_store(monkeypatch):
    dev = _dev()
    rng = np.random.default_rng(2)
    cams = _cams(dev)
    ids, frames = _batch(rng, cams, 40)
    ref = CM.undistort_frames(GT.FramesU8.pack(frames, device=dev), cams, ids)
    monkeypatch.setattr(CM, "_CHUNK_BYTES", 1 << 20)  # several chunks, each holding whole frames
    pin = GT.FramesU8.pack(frames, pin=True)
    out = CM.undistort_frames(pin, cams, ids)
    assert not out.is_cuda and out.data.is_pinned()
    assert torch.equal(out.data, ref.data.cpu())


def test_eval_frames_use_camera_0():
    """camera_ids=None undistorts every frame with the first camera, as the reference does for its eval frames."""
    dev = _dev()
    rng = np.random.default_rng(4)
    cams = _cams(dev)
    f = [rng.integers(0, 256, (47, 61, 3), dtype=np.uint8) for _ in range(3)]
    out = CM.undistort_frames(GT.FramesU8.pack(f, device=dev), cams)
    m = cams[0].map.cpu().numpy()
    for k in range(3):
        assert np.array_equal(out.frame(k).cpu().numpy(), U.remap(f[k], m))


def test_the_shim_twin_gives_the_same_map_and_bytes():
    dev = _dev()
    import gssdf_shim as shim
    rng = np.random.default_rng(6)
    for c in _cams(dev)[:2] + _cams(dev)[4:]:
        m = shim.gssdf_undistort_map(torch.from_numpy(c.K_distorted), torch.from_numpy(c.d), c.K, c.model, c.W, c.H)
        assert m.device == dev and torch.equal(m, c.map)
        f = torch.from_numpy(np.stack([_texture(rng, c.H, c.W), rng.integers(0, 256, (c.H, c.W, 3), dtype=np.uint8)])).to(dev)
        assert torch.equal(shim.gssdf_undistort(f, m), CM.undistort_frames(f, c))
        assert torch.equal(shim.gssdf_undistort(f[1], m), CM.undistort_frames(f[1:], c)[0])
    with pytest.raises(RuntimeError):  # TORCH_CHECK: not the map's size
        shim.gssdf_undistort(torch.zeros(5, 4, 3, dtype=torch.uint8, device=dev), m)
    with pytest.raises(ValueError):  # GSSDF_EINVAL: unknown model
        shim.gssdf_undistort_map(torch.eye(3), torch.zeros(4), torch.eye(3), 2, 8, 6)


# ---- training through a distorted camera ---------------------------------------------------------------------------------------------
TW, TH = 160, 120
K_D = _K(0.5 * TW, 0.5 * TW, (TW - 1) / 2.0, (TH - 1) / 2.0)  # the distorted camera: focal W / 2 as the box-room tests use
D_D = np.array([-0.2, 0.04, 0.0008, -0.0006, 0.0], np.float32)  # barrel, radial-tangential (model 0)
WIDE = (4 * TW, 4 * TH, 1.0 * TW)  # the wide pinhole the scene is rendered at before it is resampled: W, H, focal (|x| <= 2, |y| <= 1.5)


def _distorted_frames(c2w):
    """The box room as the distorted camera sees it: each distorted pixel's ray, (x, y) with distort(x, y) = K_D^-1 (j, i), read
    bilinearly from a render at the wide pinhole; quantised to 8 bits."""
    dev = _dev()
    Ww, Hw, fw = WIDE
    wide = S.box_room_color(c2w.to(dev), fw, fw, (Ww - 1) / 2.0, (Hw - 1) / 2.0, Ww, Hw)  # [B,Hw,Ww,3]
    k1, k2, p1, p2, _ = (float(v) for v in D_D)
    j = torch.arange(TW, dtype=torch.float64, device=dev)[None, :].expand(TH, TW)
    i = torch.arange(TH, dtype=torch.float64, device=dev)[:, None].expand(TH, TW)
    xd, yd = (j - float(K_D[0, 2])) / float(K_D[0, 0]), (i - float(K_D[1, 2])) / float(K_D[1, 1])
    x, y = xd.clone(), yd.clone()
    for _ in range(60):  # fixed point x = (xd - tangential(x)) / radial(x); a contraction for this barrel
        r2 = x * x + y * y
        rad = 1 + k1 * r2 + k2 * r2 * r2
        x, y = (xd - (2 * p1 * x * y + p2 * (r2 + 2 * x * x))) / rad, (yd - (p1 * (r2 + 2 * y * y) + 2 * p2 * x * y)) / rad
    r2 = x * x + y * y
    rad = 1 + k1 * r2 + k2 * r2 * r2
    assert float((x * rad + 2 * p1 * x * y + p2 * (r2 + 2 * x * x) - xd).abs().max()) < 1e-9
    assert float(x.abs().max()) < 2.0 and float(y.abs().max()) < 1.5
    grid = torch.stack([(fw * x + (Ww - 1) / 2.0) / (Ww - 1) * 2 - 1, (fw * y + (Hw - 1) / 2.0) / (Hw - 1) * 2 - 1], -1).float()
    img = torch.nn.functional.grid_sample(wide.permute(0, 3, 1, 2), grid[None].expand(len(c2w), TH, TW, 2), mode="bilinear",
                                          align_corners=True).permute(0, 2, 3, 1)
    return (img * 255 + 0.5).floor().clamp(0, 255).to(torch.uint8).contiguous()


def _train(room, seed, K, store, c2w):
    S_ = _sdf_trainer(room, 200, seed=seed, outlier_remove=True)
    sp = _splats(room, S_, 1)
    fr = room["frame"]
    G = GT.GsTrainer(S_, sp, c2w, torch.as_tensor(K), store, capacity=32 * sp["anchors"].shape[0], spatial_scale=0.5 * fr["inner_map_size"],
                     gs_iter_step=2000, sh_degree=1, outlier_remove=True, refine_gs_struct_start_iter=1000,
                     densify=dict(refine_start_iter=200, refine_every=100), sh_degree_interval=500)
    G.run()
    return G.state()


# measured on an H100 80GB HBM3 at 700 W: 34.0 dB undistorted, 21.8 dB distorted (DESIGN 7r); the bar asks for half that margin
MARGIN_MIN = 6.0


def test_undistorted_frames_train_better_than_distorted(room):
    """40 training views of the box room through the distorted camera K_D, D_D (rendered at a wide pinhole and resampled), then two runs
    of SdfTrainer (200 iterations) -> neural_gs_init -> GsTrainer (2000 joint iterations, SH degree 1): one on the frames undistorted by
    undistort_frames with set_distortion's new K, one on the distorted frames with the raw K, as a user without undistortion trains.
    Both render 12 held-out poses at the new K against the box room's pinhole ground truth there."""
    dev = _dev()
    c2w = _poses(52, 9)
    u = CM.Undistortion(TW, TH, K_D, D_D, 0, device=dev)
    dist = GT.FramesU8(_distorted_frames(c2w[:40]).reshape(-1), [(TW, TH)] * 40)
    undist = CM.undistort_frames(dist, u)
    nK = u.K.numpy()
    vms = torch.linalg.inv(c2w[40:].to(torch.float64)).to(torch.float32)
    gts = S.box_room_color(c2w[40:].to(dev), float(nK[0, 0]), float(nK[1, 1]), float(nK[0, 2]), float(nK[1, 2]), TW, TH)
    psnr = {}
    for tag, K, store in (("undistorted", u.K, undist), ("distorted", K_D, dist)):
        st = _train(room, 5, K, store, c2w[:40].contiguous())
        renders = torch.stack([st["render"](vm, camera=(TW, TH, u.K)) for vm in vms])
        full, _ = MT.eval_render(renders.clamp(0, 1), gts, [f"{i}.png" for i in range(12)])
        psnr[tag] = full["PSNR"]
    print(f"held-out PSNR at the new K: {psnr}, margin {psnr['undistorted'] - psnr['distorted']:.2f} dB")
    assert psnr["undistorted"] > psnr["distorted"] + MARGIN_MIN, psnr
