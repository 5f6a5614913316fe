"""Training the splats on frames of several cameras on the GPU (DESIGN 7q): gssdf_frames_u8_expand against the numpy fp32 product, a
joint step inside a renderer allocated for larger frames against a renderer allocated at exactly the step's size (stale pixels from a
larger step present), one camera given as [T,3,3] + a frame list against today's [3,3] + [T,H,W,3] call, 8-bit frames (device and
pinned) against the same frames expanded on the host, the densifier's pinned radii normaliser against the fp64 arbiter, and the box room
trained end to end on three cameras of different intrinsics and sizes.

The renders (projection, tile lists, raster images, post-ops) and the statistics they decide (visible count, radii, counts) are
deterministic and compared bit for bit. The visibilities, the loss, the gradients and what Adam makes of them accumulate with float
atomics, so they are compared against the spread of two runs of the reference configuration from the same state, as
tests/test_gpu_gs_train.py does."""
import ctypes

import numpy as np
import pytest
import torch

import densify_oracle as A
import gs_train_replay as RP
from gssdf_b200 import cabi
from gssdf_b200 import gstrain as GT
from gssdf_b200 import mesh as ME
from gssdf_b200 import metrics as MT
from gssdf_b200 import scene as S
from test_gpu_gs_train import SHRUNK, _poses, _sdf_trainer, _splats, room  # noqa: F401  (room: the module fixture)

pytestmark = pytest.mark.gpu
f32 = np.float32


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _K(W, H, f_mult=0.5, dx=0.0):
    """A pinhole of focal f_mult * W with the principal point dx pixels off the centre."""
    return torch.tensor([[f_mult * W, 0, (W - 1) / 2.0 + dx], [0, f_mult * W, (H - 1) / 2.0 - dx], [0, 0, 1.0]], dtype=torch.float32)


def _shared(room):
    """One SdfTrainer and its splats for the trainers below that freeze the SDF (detach_sdf_grad: they only read it)."""
    if "S_" not in room:
        room["S_"] = _sdf_trainer(room, 200, seed=3)
        room["sp"] = _splats(room, room["S_"], 1)
    return room["S_"], room["sp"]


def _restore(G, snap):
    """gs_train_replay.restore of a snapshot another trainer of the same layout took, keeping G's own lazy-SH stamp array."""
    last = G.T.sh_replay.s.last
    RP.restore(G, snap)
    G.T.sh_replay.s.last = last


def _assert_within_spread(label, got, want, other):
    """got against want, with `other` a second run of want's configuration from the same state. Float-atomic sums differ from run to run
    in their last bits, and a few entries jump: a sum that cancels to near 0 can change sign, which Adam's first steps turn into a move
    of 2 lr (m / (sqrt(v) + 1e-15) is +-1 there), and a visibility at the coupling gate's threshold switches a splat's SDF term on or
    off. So every entry must lie within 8x the two runs' largest difference (at least 1e-6 of the largest |want|), except at most one
    in 10 000; an input that differs moves far more entries than that."""
    fin = torch.isfinite(want)  # split rows carry a log-scale of -inf (neural_gaussian.cpp's log(0)): those must match exactly
    for t in (got, other):
        assert torch.equal(torch.isfinite(t), fin) and torch.equal(t[~fin].nan_to_num(), want[~fin].nan_to_num()), label
    got, want, other = got[fin], want[fin], other[fin]
    d = (got - want).abs()
    tol = 8 * max(float((other - want).abs().max()), 1e-6 * float(want.abs().max()))
    n_off = int((d > tol).sum())
    print(f"{label}: max |err| {float(d.max()):.3e}, tolerance {tol:.3e}, {n_off} / {want.numel()} entries beyond it")
    assert n_off <= want.numel() // 10000, (label, n_off, float(d.max()), tol)


def _recording_cabi(monkeypatch):
    """Replaces every entry point of cabi with a recorder of (name, arguments) in front of it; returns the list the calls go to. Tensors
    are recorded by dtype and shape, and a camera's K [.,3,3] or pose [.,4,4] also by its values; device pointers passed as ints by a
    placeholder. Two trainers that make the same launches with the same sizes, scalars, cameras and poses leave equal records."""
    calls = []

    def norm(v):
        if isinstance(v, torch.Tensor):
            cam = v.dim() >= 2 and tuple(v.shape[-2:]) in ((3, 3), (4, 4)) and v.numel() <= 16
            return (str(v.dtype), tuple(v.shape), tuple(v.flatten().tolist()) if cam else None)
        if isinstance(v, dict):
            return tuple((k, norm(x)) for k, x in v.items())
        if isinstance(v, (list, tuple)):
            return tuple(norm(x) for x in v)
        if isinstance(v, bool) or v is None or isinstance(v, (float, str)):
            return v
        if isinstance(v, int):
            return "ptr" if v > 1 << 32 else v
        return type(v).__name__

    for name in dir(cabi):
        fn = getattr(cabi, name)
        if callable(fn) and getattr(fn, "__module__", None) == cabi.__name__ and not isinstance(fn, type) and not name.startswith("_"):
            def rec(*a, _fn=fn, _name=name, **kw):
                calls.append((_name, norm(a), norm(kw)))
                return _fn(*a, **kw)
            monkeypatch.setattr(cabi, name, rec)
    return calls


def _frames(c2w, cams):
    """Box-room colour frames [H_i,W_i,3] of the poses, frame i seen by camera cams[i] = (W, H, K)."""
    out = []
    for i, (W, H, K) in enumerate(cams):
        out.append(S.box_room_color(c2w[i:i + 1].to(_dev()), float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]), W, H)[0])
    return out


# ---- the expansion kernel -----------------------------------------------------------------------------------------------------------
def test_u8_expand_is_the_fp32_product():
    """Every byte value in every channel, frames of odd sizes at odd offsets: gt == fl(x * fl(1/255)) bit for bit, channel 3 == 0, nothing
    past the frame written."""
    dev = _dev()
    rng = np.random.default_rng(0)
    inv = f32(1.0) / f32(255.0)
    sizes = [(1, 1), (17, 5), (256, 1), (33, 19), (255, 3)]
    frames = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for w, h in sizes]
    frames[2][0, :, 0] = np.arange(256)
    frames[2][0, :, 1] = np.arange(256)[::-1]
    frames[2][0, :, 2] = np.roll(np.arange(256), 7)
    st = GT.FramesU8.pack(frames, device=dev)
    assert st.offsets[1:] == np.cumsum([3 * w * h for w, h in sizes]).tolist()
    for i, (w, h) in enumerate(sizes):
        gt = torch.full((h * w * 4 + 8,), 7.0, dtype=torch.float32, device=dev)
        cabi.frames_u8_expand(st.data, st.offsets[i], w, h, gt)
        g = gt.cpu().numpy()
        want = frames[i].astype(f32) * inv
        got = g[:h * w * 4].reshape(h, w, 4)
        assert np.array_equal(got[..., :3].view(np.uint32), want.view(np.uint32)), (w, h)
        assert (got[..., 3] == 0).all() and (g[h * w * 4:] == 7.0).all()
        assert np.array_equal(st.frame(i).cpu().numpy(), frames[i])
    vals = np.arange(256, dtype=f32) * inv
    assert len(np.unique(vals)) == 256 and vals[255] == f32(1.0)
    with pytest.raises(ValueError, match="does not fit"):
        cabi.frames_u8_expand(st.data, st.offsets[-1] - 2, 1, 1, torch.zeros(4, device=dev))
    with pytest.raises(ValueError, match="bytes"):
        GT.FramesU8(st.data[:-1].clone(), sizes)


# ---- one step inside a larger allocation --------------------------------------------------------------------------------------------
def _trainer(room, S_, sp, sizes, mask=None, bck_color=0, depth_type=0, scale2d=True):
    """A GsTrainer over one frame per size (poses and pixels are placeholders: the steps below bring their own), SH degree 1, SDF frozen."""
    n = len(sizes)
    cams = [(w, h, _K(w, h)) for w, h in sizes]
    imgs = [torch.zeros(h, w, 3, device=_dev()) for w, h in sizes]
    Ks = torch.stack([c[2] for c in cams])
    fr = room["frame"]
    return GT.GsTrainer(S_, sp, torch.eye(4).repeat(n, 1, 1), Ks, imgs, capacity=sp["anchors"].shape[0], spatial_scale=0.5 * fr["inner_map_size"],
                        gs_iter_step=10, sh_degree=1, detach_sdf_grad=True, bck_color=bck_color, mask=mask, depth_type=depth_type,
                        densify=dict(refine_scale2d_stop_iter=5 if scale2d else 0))


def _joint(G, vm, K, img, randn, bg, normal_w, mask=None):
    """One joint step of GsTrainer's at img's size (no SDF ray stage: the SDF is frozen), Adam, and the densifier's statistics."""
    H, W = img.shape[:2]
    G.set_frame(W, H)
    if mask is not None:
        G.T.set_frame(W, H, mask=mask)
    G.gt[0, ..., :3].copy_(img)
    G.randns.copy_(randn)
    if G.T.bg is not None:
        G.T.bg.copy_(bg[:H * W * 3].view(1, H, W, 3))
    G.T.normal_w = normal_w
    G.T.train_step(vm, K, G.gt, None, None, G.randns)
    R = G.T.R
    nnz = min(int(R.counts[0]), R.cap)
    out = dict(loss=R.loss.clone(), grad=G.T.flat_grad.clone(), counts=R.counts[:2].clone(), vis=R.r["visibilities"][:nnz].clone())
    for k in ("render_colors", "render_depths", "render_alphas", "render_normals", "render_median", "last_ids", "median_ids"):
        out[k] = R.r[k].clone()
    out["out_colors"], out["out_normals"], out["v_out_normals"] = R.out_colors.clone(), R.out_normals.clone(), R.v_out_normals.clone()
    G.T.adam_clocks(sdf=False)
    G.T.flat_grad[G.T.t0:].zero_()  # [C]'s SDF gradient: no optimiser group consumes it (GsTrainer.step with detach_sdf_grad)
    G.D.update_state()
    out.update({"st_" + k: v.clone() for k, v in G.D.state.items()})
    out["params"], out["m"], out["v"] = G.T.params.clone(), G.T.exp_avg.clone(), G.T.exp_avg_sq.clone()
    return out


EXACT = ("counts", "render_colors", "render_depths", "render_alphas", "render_normals", "render_median", "last_ids", "median_ids",
         "out_colors", "out_normals", "st_count", "st_radii")
SPREAD = ("loss", "vis", "grad", "st_vis", "st_grad2d", "params", "m", "v")  # the visibilities are float-atomic sums over tiles


def _copy_state(dst, src):
    """Everything a joint step reads that is not a per-pixel buffer: parameters, moments, clocks, the lazy-SH stamps, the rates, the
    densifier's statistics and its radii normaliser."""
    T, U = dst.T, src.T
    for a in ("_params", "_exp_avg", "_exp_avg_sq", "anchors_buf", "flat_grad", "table_half", "mlp_packed", "sh_last"):
        getattr(T, a).copy_(getattr(U, a))
    last = T.sh_replay.s.last  # the replay window's scalars, with dst's own stamp array
    ctypes.memmove(ctypes.addressof(T.sh_replay.s), ctypes.addressof(U.sh_replay.s), ctypes.sizeof(U.sh_replay.s))
    T.sh_replay.s.last = last
    T.t_splat, T.t_sh, T.t_sdf, T.lr, T.sdf_lr, T._sh_stale = U.t_splat, U.t_sh, U.t_sdf, list(U.lr), U.sdf_lr, U._sh_stale
    T.R.sh_degree = U.R.sh_degree
    T.set_live(U.N_live)
    for k, v in src.D.state.items():
        dst.D.state[k].copy_(v)
    dst.D.pin_image_size, dst.D.image_size = src.D.pin_image_size, src.D.image_size

# (size of the compared step, larger size stepped before it, bck_color, mask, depth_type, normal term in the large / compared step)
CASES = [
    ((157, 93), (200, 112), 0, False, 0, True, True),      # not multiples of 16
    ((111, 127), (128, 128), 1, True, 1, True, True),      # 56 tiles (tile_n_bits 6) after 64 (tile_n_bits 7)
    ((144, 112), (160, 100), 2, False, 1, True, False),    # 63 tiles (6 bits) after 70 (7 bits); the normal cotangents go stale
    ((157, 93), (200, 112), 2, True, 0, True, False),
    ((111, 127), (128, 128), 0, False, 1, False, True),
]


@pytest.mark.parametrize("case", CASES, ids=[f"{c[0][0]}x{c[0][1]}-after-{c[1][0]}x{c[1][1]}-bck{c[2]}-mask{int(c[3])}-d{c[4]}" for c in CASES])
def test_step_inside_a_larger_allocation(room, case):
    """A trainer allocated for the compared frame size (its first frame) and a larger one runs a step at the larger size, then one at the
    compared size; two trainers allocated at exactly the compared size run the same second step from the same state. Everything the step
    computes deterministically is bit-identical; the float-atomic results lie within the two exact trainers' spread. Where the normal
    term is on at the larger size only, a third step at the larger size follows, against trainers allocated at exactly that size. (144x112
    has more pixels than 160x100 but fewer tiles: the storage holds the larger of each.)"""
    (W, H), (Wb, Hb), bck, use_mask, depth_type, nw_big, nw = case
    dev = _dev()
    S_, sp = _shared(room)
    gen = torch.Generator().manual_seed(hash(case) % 2 ** 31)
    mask = (torch.rand(H, W, generator=gen) > 0.2).to(dev) if use_mask else None
    big = _trainer(room, S_, sp, [(W, H), (Wb, Hb)], bck_color=bck, depth_type=depth_type)
    refs = [_trainer(room, S_, sp, [(W, H)], mask=mask, bck_color=bck, depth_type=depth_type) for _ in range(2)]
    assert big.multi_size and big.D.pin_image_size and not refs[0].multi_size
    assert big.T.R.max_pixels == max(W * H, Wb * Hb) and refs[0].T.R.max_pixels == W * H
    c2w = _poses(2, 21)
    vms = torch.linalg.inv(c2w.to(torch.float64)).to(torch.float32).to(dev).contiguous()
    K, Kb = _K(W, H).reshape(1, 3, 3).to(dev), _K(Wb, Hb, 0.6, 3.0).reshape(1, 3, 3).to(dev)
    img = _frames(c2w[:1], [(W, H, _K(W, H))])[0]
    img_b = _frames(c2w[1:], [(Wb, Hb, Kb[0].cpu())])[0]
    randn = [torch.randn(big.randns.shape, generator=gen).to(dev) for _ in range(2)]
    bg = [torch.rand(max(W * H, Wb * Hb) * 3, generator=gen).to(dev) for _ in range(2)]
    # the larger step fills every buffer past the compared frame with live values
    _joint(big, vms[1:2], Kb, img_b, randn[0], bg[0], 0.01 if nw_big else 0.0)
    # ...which the exact trainers reach without it: the same parameters, moments and clocks, the larger step's statistics
    for G in refs:
        _copy_state(G, big)
    got = _joint(big, vms[0:1], K, img, randn[1], bg[1], 0.01 if nw else 0.0, mask=mask)
    want = [_joint(G, vms[0:1], K, img, randn[1], bg[1], 0.01 if nw else 0.0) for G in refs]
    torch.cuda.synchronize()
    assert int(got["counts"][0]) > 100
    for k in EXACT:
        if got.get(k) is None:
            continue
        assert got[k].shape == want[0][k].shape and torch.equal(got[k], want[0][k]), k
    for k in SPREAD:
        _assert_within_spread(f"{case[0]} {k}", got[k], want[0][k], want[1][k])
    if nw_big and not nw:
        # back at the larger size without the normal term: the normal cotangent the first step wrote past the smaller frame was cleared
        # with the rest of the storage, so the step equals one on trainers allocated at exactly the larger size
        refs_b = [_trainer(room, S_, sp, [(Wb, Hb)], bck_color=bck, depth_type=depth_type) for _ in range(2)]
        for G in refs_b:
            _copy_state(G, big)
        big.T.mask = None  # the image mask belongs to the smaller frame
        got = _joint(big, vms[1:2], Kb, img_b, randn[0], bg[0], 0.0)
        want = [_joint(G, vms[1:2], Kb, img_b, randn[0], bg[0], 0.0) for G in refs_b]
        assert torch.equal(big.T.R.v_out_normals, want[0]["v_out_normals"]) and not big.T.R.v_out_normals.any()
        for k in EXACT:
            assert torch.equal(got[k], want[0][k]), ("larger again", k)
        for k in SPREAD:
            _assert_within_spread(f"{(Wb, Hb)} again {k}", got[k], want[0][k], want[1][k])


def test_set_frame_rejects_frames_past_the_storage(room):
    S_, sp = _shared(room)
    G = _trainer(room, S_, sp, [(100, 60), (64, 64)])
    R = G.T.R
    assert (R.max_pixels, R.max_tiles) == (6000, 28)  # 7 x 4 tiles, 4 x 4 tiles
    R.set_frame(112, 48)  # 5376 pixels, 7 x 3 tiles: fits
    assert R.out_colors.shape == (1, 48, 112, 4) and R.offsets.shape == (1, 3, 7) and R.out_colors.is_contiguous()
    assert R.out_colors.data_ptr() == R._pix[(None, "out_colors")].data_ptr()
    for w, h in ((101, 60), (60, 101), (16 * 29, 1)):  # 6060 pixels twice; 464 pixels in 29 tiles
        with pytest.raises(ValueError, match="does not fit"):
            R.set_frame(w, h)
    with pytest.raises(ValueError, match="image mask"):
        G.T.mask = torch.ones(60, 100, 3, dtype=torch.uint8, device=_dev())
        G.T.set_frame(64, 64)


# ---- one camera through the new arguments -------------------------------------------------------------------------------------------
def test_one_camera_as_a_table_equals_todays_call(room, monkeypatch):
    """K [T,3,3] of equal rows and the frames as a list train as K [3,3] and [T,H,W,3] do: 40 joint iterations (shrunk constants: growth
    at 4, 8, 12, 16, an opacity reset, invisible prunes, an outlier removal) run in lockstep, each from the same state. Both make the
    same library calls with the same sizes, scalars, cameras and poses, on bit-identical ground truth; everything the host-driven replay
    test pins bit for bit agrees bit for bit; parameters and moments lie within the spread of two runs of today's call."""
    S_ = _sdf_trainer(room, 200, seed=12, outlier_remove=True)
    sp = _splats(room, S_, 1)
    c2w = _poses(6, 22)
    W, H = 160, 120
    K = _K(W, H)
    imgs = S.box_room_color(c2w.to(_dev()), float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]), W, H)
    fr = room["frame"]
    kw = dict(capacity=8 * sp["anchors"].shape[0], spatial_scale=0.5 * fr["inner_map_size"], gs_iter_step=40, sh_degree=1, **SHRUNK)
    A_ = GT.GsTrainer(S_, sp, c2w, K, imgs, **kw)
    B_ = GT.GsTrainer(S_, sp, c2w, K.repeat(6, 1, 1), [imgs[i].clone() for i in range(6)], **kw)
    assert not B_.multi_size and not B_.D.pin_image_size and B_.T.R.max_pixels == W * H
    A_.run_color_init()
    _restore(B_, RP.snapshot(A_))
    rs = S_.rs

    def capture(G):
        n = int(rs.counts[0])
        T = G.T
        return dict(counts=rs.counts[:3].tolist(), xyz=rs.xyz[:n].clone(), state=S_.adapt.tolist(), N_live=T.N_live, log=list(G.D.log),
                    N=S_.N, sh=T.R.sh_degree, p=T.params.clone(), m=T.exp_avg.clone(), v=T.exp_avg_sq.clone(),
                    out=T.R.out_colors.clone(), loss=float(G.h_loss[G.done - 1]))
    A_.start_rates()
    B_.start_rates()
    calls = _recording_cabi(monkeypatch)
    for i in range(40):
        snap = RP.snapshot(A_)
        A_.step(i)
        a = capture(A_)
        RP.restore(A_, snap)
        del calls[:]
        A_.step(i)
        b = capture(A_)
        calls_a, calls[:] = list(calls), []
        gt_a, K_a = A_.gt.clone(), A_.K_cur.clone()
        _restore(B_, snap)
        del calls[:]
        B_.step(i)
        d = capture(B_)
        assert calls == calls_a and len(calls) > 20, i
        assert torch.equal(B_.gt, gt_a) and torch.equal(B_.K_cur, K_a), i
        for k in ("counts", "state", "N_live", "log", "N", "sh"):
            assert d[k] == a[k] == b[k], (i, k, d[k], a[k])
        assert torch.equal(d["xyz"], a["xyz"]) and torch.equal(d["out"], a["out"]), i
        for k in ("p", "m", "v"):
            _assert_within_spread(f"{i} {k}", d[k], a[k], b[k])
        _restore(A_, RP.snapshot(B_))
    assert [e[0] for e in B_.D.log][:2] == [4, 8]


# ---- 8-bit frames -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pinned", [False, True], ids=["device", "pinned"])
def test_u8_frames_train_as_host_expanded_frames(room, pinned):
    """Colour initialisation + 6 joint iterations on an 8-bit store of two sizes against the same frames expanded on the host into float
    frames: every ground truth the trainer loads is bit-identical, and so is everything the host-driven replay test pins."""
    S_, sp = _shared(room)
    c2w = _poses(4, 23)
    cams = [(160, 120, _K(160, 120)), (131, 77, _K(131, 77, 0.7, 2.0))] * 2
    u8 = [(f * 255).round().clamp(0, 255).to(torch.uint8).cpu() for f in _frames(c2w, cams)]
    host = [(t.numpy().astype(f32) * (f32(1.0) / f32(255.0))) for t in u8]
    fr = room["frame"]
    kw = dict(capacity=sp["anchors"].shape[0], spatial_scale=0.5 * fr["inner_map_size"], gs_iter_step=6, sh_degree=1, detach_sdf_grad=True)
    Ks = torch.stack([c[2] for c in cams])
    st = GT.FramesU8.pack(u8, device=None if pinned else _dev(), pin=pinned)
    G8 = GT.GsTrainer(S_, sp, c2w, Ks, st, **kw)
    GF = GT.GsTrainer(S_, sp, c2w, Ks, [torch.from_numpy(h).to(_dev()) for h in host], **kw)
    assert G8.multi_size and GF.multi_size and (G8._stage_store is not None) == pinned
    for i in range(4):
        G8.load_frame(i)
        GF.load_frame(i)
        assert torch.equal(G8.gt, GF.gt) and G8.gt.shape == (1, cams[i][1], cams[i][0], 4), i
        assert torch.equal(G8.K_cur, GF.K_cur) and torch.equal(G8.K_cur[0], Ks[i].to(_dev()))
    G8.run_color_init()
    GF.run_color_init()
    G8.start_rates()
    GF.start_rates()
    for i in range(6):
        G8.step(i)
        GF.step(i)
        assert torch.equal(G8.gt, GF.gt), i
    torch.cuda.synchronize()
    h8, hf = G8.histories(), GF.histories()
    assert np.allclose(h8["color_loss"], hf["color_loss"], rtol=1e-4) and np.allclose(h8["loss"], hf["loss"], rtol=1e-3)
    assert np.array_equal(h8["n_live"], hf["n_live"])


# ---- the densifier's radii normaliser -----------------------------------------------------------------------------------------------
def test_densify_radii_normaliser_is_the_first_frames(room):
    """Two frame sizes, refine_scale2d_stop_iter > 0: after each of four steps (sizes alternating, the smaller first) the statistics match
    the fp64 arbiter: grad2d scaled by each frame's own width and height, radii divided by max(W, H) of the first frame."""
    S_, sp = _shared(room)
    sizes = [(96, 72), (200, 112)]
    G = _trainer(room, S_, sp, sizes)
    D, R = G.D, G.T.R
    c2w = _poses(4, 24)
    vms = torch.linalg.inv(c2w.to(torch.float64)).to(torch.float32).to(_dev()).contiguous()
    N = G.T.N_live
    state = {k: np.zeros(N, f32) for k in ("grad2d", "count", "vis", "radii")}
    image_size = max(sizes[0])
    for i in range(4):
        W, H = sizes[i % 2]
        K = _K(W, H).reshape(1, 3, 3).to(_dev())
        G.set_frame(W, H)
        G.gt[0, ..., :3].copy_(_frames(c2w[i:i + 1], [(W, H, _K(W, H))])[0])
        G.randns.normal_(generator=G.gen)
        G.T.train_step(vms[i:i + 1], K, G.gt, None, None, G.randns)
        nnz = min(int(R.counts[0]), R.cap)
        gid, vd = R.p["gaussian_ids"][:nnz].cpu().numpy(), R.g["v_densify"][:nnz].cpu().numpy()
        vis, rad = R.r["visibilities"][:nnz, 0].cpu().numpy(), R.p["radii"][:nnz].cpu().numpy()
        D.update_state()
        G.T.flat_grad.zero_()
        prev = dict(state)
        want, scale = A.update_state(state, gid, vd, vis, rad, W, H, 1)
        want_r, _ = A.update_state(state, gid, vd, vis, rad, image_size, image_size, 1)
        want["radii"] = want_r["radii"]
        assert D.image_size == float(image_size)
        for k in ("grad2d", "count", "vis", "radii"):
            got = D.state[k][:N].cpu().numpy()
            bad = A.off_bar(got.astype(np.float64), want[k], scale[k])
            assert not bad.any(), (i, k, int(bad.sum()))
            state[k] = got
        assert (state["radii"] > 0).any()
    # the last step's frame is the larger one: its own max(W, H) would have given other radii
    assert not np.array_equal(A.update_state(prev, gid, vd, vis, rad, 200, 112, 1)[0]["radii"], want["radii"])


# ---- the box room on three cameras ---------------------------------------------------------------------------------------------------
CAMS3 = [(160, 120, 0.5, 0.0), (128, 96, 0.62, 4.0), (200, 112, 0.45, -3.0)]
# measured on an H100 80GB HBM3 at 700 W: 26.6, 29.0 and 28.7 dB (the single-camera test's 12 poses at 160x120: 28.7 dB); the bar
# leaves 3 dB under the weakest camera
PSNR_MIN = 23.5


def test_end_to_end_on_three_cameras(room):
    """SdfTrainer (200 iterations) -> neural_gs_init -> GsTrainer (colour init + 2000 joint iterations, SH degree 1) over 60 training
    views, 20 per camera, on three cameras that differ in focal length, principal point and size; the PSNR of each camera over the 12
    held-out poses of the single-camera test rendered at that camera, and the mesh of the jointly trained SDF. Measured on an H100: see
    DESIGN 7q."""
    S_ = _sdf_trainer(room, 200, seed=5, outlier_remove=True)
    sp = _splats(room, S_, 1)
    c2w = _poses(72, 9)
    cams = [(w, h, _K(w, h, f, dx)) for w, h, f, dx in CAMS3]
    frame_cam = [i % 3 for i in range(60)]
    imgs = _frames(c2w[:60], [cams[c] for c in frame_cam])
    fr = room["frame"]
    G = GT.GsTrainer(S_, sp, c2w[:60].contiguous(), torch.stack([cams[c][2] for c in frame_cam]), imgs,
                     capacity=32 * sp["anchors"].shape[0], spatial_scale=0.5 * fr["inner_map_size"], gs_iter_step=2000, sh_degree=1,
                     outlier_remove=True, refine_gs_struct_start_iter=1000, densify=dict(refine_start_iter=200, refine_every=100),
                     sh_degree_interval=500)
    G.run()
    h = G.histories()  # raises on a sampler overflow
    st = G.state()
    vms = torch.linalg.inv(c2w[60:].to(torch.float64)).to(torch.float32)
    psnr = {}
    for W, H, K in cams:
        renders = torch.stack([st["render"](vm, camera=(W, H, K)) for vm in vms])
        gts = _frames(c2w[60:], [(W, H, K)] * 12)
        full, _ = MT.eval_render(renders.clamp(0, 1), torch.stack(gts), [f"{i}.png" for i in range(12)])
        psnr[(W, H)] = full["PSNR"]
    v, f, _ = ME.meshing(room["tree"], st["net"], room["margin"][0], room["margin"][1], 0.025)
    gt = S.box_wall_points(0.01)
    mm = ME.eval_mesh(v, f, torch.from_numpy(gt).to(_dev()), mesh_sample_point=1_000_000, gt_bbx_mask_on=False)
    print(f"held-out PSNR per camera {psnr}; mesh {mm}; N_live {h['n_live'][-1]}; events {len(h['densify_events'])}; "
          f"loss last {h['loss'][-3:]}")
    assert G.D.image_size in (160.0, 128.0, 200.0)  # max(W, H) of the first joint iteration's frame
    for c, p in psnr.items():
        assert p > PSNR_MIN, (c, p)
    # the single-camera run's band (tests/test_gpu_gs_train.py::test_end_to_end_on_the_box_room)
    assert mm["MAE_accuracy (cm)"] < 1.0 and mm["MAE_completeness (cm)"] < 1.0 and mm["F-score (%)"] > 97.0
