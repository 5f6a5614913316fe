"""The joint stage on the GPU (gstrain.GsTrainer, DESIGN 7o): gssdf_adam_step_clocks against torch.optim.Adam with per-parameter step
counts, gssdf_adam_step against outputs recorded before the per-group clocks existed, a short run with every schedule event, every
iteration against a host-driven replay in the reference's order (with and without an injected NaN), where the iterations synchronise,
pinned against device frames, the argument errors, and the whole pipeline on the box room (SdfTrainer -> neural_gs_init -> GsTrainer ->
held-out PSNR and mesh metrics)."""
import math
import os

import numpy as np
import pytest
import torch

from gssdf_b200 import cabi
from gssdf_b200 import gs_init as GI
from gssdf_b200 import gstrain as GT
from gssdf_b200 import mesh as ME
from gssdf_b200 import metrics as MT
from gssdf_b200 import nsdf as NS
from gssdf_b200 import octree as OT
from gssdf_b200 import scene as S
from gssdf_b200 import sdf as SD
from gssdf_b200.render import sh_sweep_step

pytestmark = pytest.mark.gpu
f32 = np.float32
LEAF, BCE_SIGMA = 0.05, 0.01
W, H = 160, 120
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "adam_legacy.npz")


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


# ---- the optimiser -------------------------------------------------------------------------------------------------------------------
def test_adam_step_is_bit_identical_to_the_recorded_outputs():
    """gssdf_adam_step (dense, half-shadow and lazy row groups, 70 steps across a window boundary, grad_scale 0.5 every third step) gives
    the bits the single-clock optimiser gave on the same inputs."""
    import adam_legacy_case as A
    g = np.load(GOLDEN)
    inp = {k[3:]: g[k] for k in g.files if k.startswith("in_")}
    out = A.run(inp, _dev())
    for k, v in out.items():
        assert np.array_equal(v.view(np.uint8), g["out_" + k].view(np.uint8)), k
    # the clocks entry with every group at the same step is the same update
    clk = A.run(inp, _dev(), step_fn=lambda p, g_, m, v_, grp, t, **kw: cabi.adam_step_clocks(p, g_, m, v_, grp, [t] * len(grp), **kw))
    for k, v in out.items():
        assert np.array_equal(v.view(np.uint8), clk[k].view(np.uint8)), k


def test_adam_clocks_against_torch_adam_with_per_parameter_steps():
    """Three clocks as the joint stage has them: an 'SDF' group that stepped 10 times alone, SH row groups (lazy: each step visits a
    random half of the rows) that then stepped 5 times alone, then 70 steps of everything in one launch (across the 64-step window). The
    reference is torch.optim.Adam (fp32, eps 1e-15), whose per-parameter state skips a parameter without a gradient."""
    dev = _dev()
    rng = np.random.default_rng(1)
    R, w0, w1 = 300, 3, 9
    sizes = dict(sdf=2051, other=1003, dc=R * w0, rest=R * w1)
    off, o = {}, 0
    for k in ("other", "dc", "rest", "sdf"):
        off[k] = o
        o += sizes[k] + (sizes[k] % 2)
    n = o
    lrs = dict(sdf=5e-3, other=1e-3, dc=2.5e-3, rest=1.25e-4)
    p0 = rng.standard_normal(n).astype(f32)
    p, m, v, g = (torch.from_numpy(p0).to(dev), torch.zeros(n, device=dev), torch.zeros(n, device=dev), torch.zeros(n, device=dev))
    tp = {k: torch.nn.Parameter(torch.from_numpy(p0[off[k]:off[k] + sizes[k]].copy()).to(dev)) for k in sizes}
    opt = torch.optim.Adam([dict(params=[tp[k]], lr=lrs[k]) for k in sizes], eps=1e-15)
    last = torch.zeros(R, dtype=torch.int32, device=dev)
    replay = cabi.AdamReplay(last)
    counts = torch.zeros(cabi.COUNTS_INTS, dtype=torch.int32, device=dev)
    grp = {k: (off[k], sizes[k], lrs[k], False, {"dc": w0, "rest": w1}.get(k, 0)) for k in sizes}
    clocks = dict(sdf=0, sh=0, other=0)

    def one(active):
        for k in tp:
            tp[k].grad = None
        g.zero_()
        if "sh" in active:
            ids = np.sort(rng.choice(R, R // 2, replace=False))
            rows = torch.zeros(R, device=dev)
            rows[torch.from_numpy(ids).to(dev)] = 1
        for k in sizes:
            if (k in ("dc", "rest") and "sh" in active) or k in active:
                gk = torch.from_numpy(rng.standard_normal(sizes[k]).astype(f32) * f32(0.01)).to(dev)
                if k in ("dc", "rest"):
                    gk = (gk.view(R, -1) * rows[:, None]).reshape(-1)
                g[off[k]:off[k] + sizes[k]] = gk
                tp[k].grad = gk.clone()
        opt.step()
        groups, steps = [], []
        for k in ("other", "dc", "rest", "sdf"):
            c = "sh" if k in ("dc", "rest") else k
            if c in active:
                groups.append(grp[k])
        for c in active:
            clocks[c] += 1
        if "sh" in active:
            replay.push(clocks["sh"], lrs["dc"], lrs["rest"])
        steps = [clocks["sh" if gg[4] else ("sdf" if gg[0] == off["sdf"] else "other")] for gg in groups]
        row = {}
        if "sh" in active and not sh_sweep_step(clocks["sh"]):
            counts[0] = len(ids)
            row = dict(row_ids=torch.from_numpy(ids).to(dev), row_count=counts, row_cap=len(ids))
        cabi.adam_step_clocks(p, g, m, v, groups, steps, replay=replay, **row)

    for _ in range(10):
        one(("sdf",))
    for _ in range(5):
        one(("sh",))
    for _ in range(70):
        one(("sdf", "sh", "other"))
    assert clocks == dict(sdf=80, sh=75, other=70)
    cabi.adam_step(p, g, m, v, [grp["dc"], grp["rest"]], clocks["sh"], replay=replay, replay_only=True)
    for k in sizes:
        got = p[off[k]:off[k] + sizes[k]]
        assert torch.allclose(got, tp[k].detach(), rtol=2e-6, atol=2e-7), (k, (got - tp[k]).abs().max().item())
        st = opt.state[tp[k]]
        assert int(st["step"]) == {"sdf": 80, "other": 70}.get(k, 75)
        # torch accumulates v as mul_(b2).addcmul_(g, g, 1 - b2): another rounding sequence, ~1e-5 relative after 80 steps
        assert torch.allclose(v[off[k]:off[k] + sizes[k]], st["exp_avg_sq"], rtol=1e-4, atol=1e-12)


def test_adam_clocks_rejects_row_groups_on_two_clocks():
    dev = _dev()
    p = torch.zeros(64, device=dev)
    replay = cabi.AdamReplay(torch.zeros(8, dtype=torch.int32, device=dev))
    replay.push(3, 1e-3, 1e-3)
    groups = [(0, 8 * 3, 1e-3, False, 3), (24, 8 * 4, 1e-3, False, 4)]
    with pytest.raises(ValueError, match="differ in step"):
        cabi.adam_step_clocks(p, p.clone(), p.clone(), p.clone(), groups, [3, 4], replay=replay)
    with pytest.raises(ValueError, match="step"):
        cabi.adam_step_clocks(p, p.clone(), p.clone(), p.clone(), groups[:1], [0], replay=replay)
    with pytest.raises(ValueError, match="steps for"):
        cabi.adam_step_clocks(p, p.clone(), p.clone(), p.clone(), groups, [3], replay=replay)


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


@pytest.fixture(scope="module")
def room():
    dev = _dev()
    pack = S.box_room_pack(dev, 120, ds_pt_num=2000, seed=0)
    tree, frame, _ = OT.build_occ_map(pack["xyz"], pack["depth"], 0.01, 100.0, 14.0, LEAF)
    pos = np.asarray(frame["origin"], f32)
    lo = tuple(float(f32(pos[k] + f32(frame["xyz_min_M"][k]))) for k in range(3))
    hi = tuple(float(f32(pos[k] + f32(frame["xyz_max_M"][k]))) for k in range(3))
    margin = (tuple(float(f32(f32(v) + f32(0.5 * LEAF))) for v in frame["xyz_min_M"]),
              tuple(float(f32(f32(v) - f32(0.5 * LEAF))) for v in frame["xyz_max_M"]))
    return dict(pack=pack, tree=tree, frame=frame, lo=lo, hi=hi, margin=margin)


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


def _recorders(G):
    """Wrap the stage's host-synchronising actions: returns a dict of the iterations at which each ran (and what it removed)."""
    rec = dict(outlier=[], invisible=[], nan=[])
    S_, D = G.sdf, G.D
    ro, pi, pn = S_.remove_outliers, D.prune_invisible_gs, D.prune_nan_gs

    def remove_outliers(i, **kw):
        n0 = S_.N
        ro(i, **kw)
        rec["outlier"].append((i, n0 - S_.N))

    def prune_invisible(it):
        n = pi(it)
        if it > 0 and it % D.num_train_data == 0:
            rec["invisible"].append((it, n))
        return n

    def prune_nan(it):
        n = pn(it)
        if n:
            rec["nan"].append((it, n))
        return n
    S_.remove_outliers, D.prune_invisible_gs, D.prune_nan_gs = remove_outliers, prune_invisible, prune_nan
    return rec


def test_short_run_hits_every_schedule_event(room):
    """20 iterations with shrunk constants: colour init over 6 frames, growth at 4 and 8, an opacity reset at 8, an invisible prune at 6,
    an SH-degree change at 5, an outlier removal at 10, the second half without callbacks."""
    S_ = _sdf_trainer(room, 200, seed=1, outlier_remove=True)
    c2w = _poses(6, 5)
    G = _gs_trainer(room, S_, (c2w, _images(c2w)), 20, **SHRUNK)
    rec = _recorders(G)
    std0 = NS.read_state(S_.adapt)
    n_rays0, n_pack0 = std0[2], S_.N
    G.run()
    torch.cuda.synchronize()
    h = G.histories()
    T = G.T
    assert (T.t_sdf, T.t_sh, T.t_splat) == (200 + 20, 6 + 20, 20)
    assert T.R.sh_degree == 1 and G.h_color.numel() == 6 and np.isfinite(h["color_loss"]).all()
    assert np.isfinite(h["loss"]).all() and np.isfinite(h["sdf_loss"]).all() and (h["n_samples"] > 0).all() and (h["vis_n"] > 0).all()
    assert [e[0] for e in h["densify_events"]] == [4, 8]
    assert [r[0] for r in rec["invisible"]] == [6] and [r[0] for r in rec["outlier"]] == [10]
    assert all(it < 10 for it, _ in rec["nan"])  # a NaN row the training produces is pruned in the first half only
    assert rec["outlier"][0][1] == n_pack0 - S_.N
    assert h["n_live"][-1] == T.N_live and len(h["n_live"]) == 20
    assert len(set(h["n_live"][10:].tolist())) == 1  # no surgery in the second half
    st = NS.read_state(S_.adapt)
    assert st[2] == n_rays0  # the joint stage never changes the ray count
    assert h["sample_std"][-1] == np.float32(st[0]) and (h["sample_std"] >= np.float32(BCE_SIGMA)).all()
    # the rates: offsets frozen at Densifier's iteration-9 rate, the others at lr * 10 * (double)0.1f
    assert T.lr[0] == GT.xyz_lr(9, 20, G.spatial_scale)
    assert T.lr[1] == GT.color_init_lr(0.001) and T.lr[4] == GT.color_init_lr(0.0025)


@pytest.mark.parametrize("nan_at", [None, 7])
def test_iterations_equal_a_host_driven_replay(room, nan_at):
    """Every joint iteration of a 20-iteration run (shrunk constants: growth at 4 and 8, opacity reset at 8, invisible prune at 6, SH
    degree change at 5, normal term from 4, outlier removal at 10) is run twice the reference's way (gs_train_replay.host_step: .item()
    reads of the sample std and the ray count, host-scalar sampler and SDF sites, .item() logging, the sample std taken in torch from the
    forward's isigma) and once by GsTrainer.step, all three from the same state. The sampler's output, the ray-site SDF variants, the
    sample std, the ray count, N_live and the densification events agree bit for bit; parameters and Adam moments agree within a few
    spreads of the two host-driven runs (float atomics in the backward). nan_at: a NaN written into one row's offsets after that
    iteration's optimiser step, which the NaN prune of the same iteration removes on both sides."""
    import gs_train_replay as RP
    S_ = _sdf_trainer(room, 200, seed=6, outlier_remove=True)
    c2w = _poses(6, 10)
    G = _gs_trainer(room, S_, (c2w, _images(c2w)), 20, **SHRUNK)
    rec = _recorders(G)
    cb = G.D.train_callback

    def train_callback(it, total):
        if it == nan_at:
            G.T.scene["raw"]["offsets"][3, 1] = float("nan")
        return cb(it, total)
    G.D.train_callback = train_callback
    G.run_color_init()
    G.start_rates()
    rs = S_.rs

    def capture():
        n = int(rs.counts[0])
        T = G.T
        return dict(counts=rs.counts[:3].tolist(), xyz=rs.xyz[:n].clone(), ray_sdf=T.ray_sdf.view(7, rs.cap)[1:, :n].clone(),
                    state=S_.adapt.tolist(), N_live=T.N_live, log=list(G.D.log), N=S_.N, sh=T.R.sh_degree,
                    p=T.params.clone(), m=T.exp_avg.clone(), v=T.exp_avg_sq.clone(), loss=float(G.h_loss[G.done - 1]))
    for i in range(20):
        snap = RP.snapshot(G)
        RP.host_step(G, i)
        a = capture()
        RP.restore(G, snap)
        RP.host_step(G, i)
        b = capture()
        RP.restore(G, snap)
        G.step(i)
        d = capture()
        for k in ("counts", "state", "N_live", "log", "N", "sh"):
            assert d[k] == a[k] == b[k], (i, k, d[k], a[k])
        for k in ("xyz", "ray_sdf"):
            assert torch.equal(d[k], a[k]), (i, k)
        for k in ("p", "m", "v"):
            spread = float((a[k] - b[k]).abs().max())
            err = float((d[k] - a[k]).abs().max())
            assert err <= 8 * max(spread, 1e-7 * float(a[k].abs().max())), (i, k, err, spread)
        assert abs(d["loss"] - a["loss"]) <= 1e-5 * abs(a["loss"]) + 2 * abs(a["loss"] - b["loss"]), i
        assert G.T.normal_w == (0.01 if i > 3 else 0.0)
    assert [e[0] for e in G.D.log] == [4, 8]
    assert 10 in [r[0] for r in rec["outlier"]] and 6 in [r[0] for r in rec["invisible"]]
    assert [r for r in rec["nan"] if r[0] == nan_at] == ([(nan_at, 1)] * 3 if nan_at is not None else [])
    n_live = G.histories()["n_live"]
    if nan_at is not None:
        assert n_live[nan_at] == n_live[nan_at - 1] - 1


def test_iterations_synchronise_only_where_the_reference_reads_back(room):
    """Under torch.cuda.set_sync_debug_mode("error"), a first half with growth, an opacity reset, invisible prunes and an outlier removal,
    and a second half, synchronise only inside the NaN prune's read, a due invisible prune, the refinement surgery and the outlier
    removal (each allowed while it runs). torch's sync detection sees the synchronising torch calls, not waits inside the C library,
    which never synchronises."""
    S_ = _sdf_trainer(room, 100, seed=2, outlier_remove=True)
    c2w = _poses(6, 6)
    G = _gs_trainer(room, S_, (c2w, _images(c2w)), 40, capacity_mult=8, **dict(SHRUNK, outlier_removal_interval=12))
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
        for i in range(1, 32):
            G.step(i)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    h = G.histories()
    assert np.isfinite(h["loss"]).all() and (h["n_samples"] > 0).all()
    assert [e[0] for e in h["densify_events"]][:2] == [4, 8]


def test_pinned_frames_match_device_frames(room):
    """Frames in pinned host memory, copied one per iteration, train as frames resident on the device: losses and parameters agree
    within the spread of the loss's and the backward's float atomics."""
    S_ = _sdf_trainer(room, 200, seed=3)
    sp = _splats(room, S_, 1)
    c2w = _poses(6, 7)
    imgs = _images(c2w)
    kw = dict(capacity=sp["anchors"].shape[0], spatial_scale=7.0, gs_iter_step=8, sh_degree=1)
    A = GT.GsTrainer(S_, sp, c2w, _K(), imgs, **kw)
    B = GT.GsTrainer(S_, sp, c2w, _K(), imgs.cpu().pin_memory(), **kw)
    A.run_color_init()
    B.run_color_init()
    torch.cuda.synchronize()
    assert torch.allclose(A.h_color, B.h_color, rtol=1e-4)
    assert torch.allclose(A.T.params, B.T.params, rtol=1e-4, atol=1e-5)


def test_argument_errors(room):
    S_ = _sdf_trainer(room, 200, seed=4)
    c2w = _poses(6, 8)
    imgs = _images(c2w)
    sp = _splats(room, S_, 1)
    n = sp["anchors"].shape[0]
    kw = dict(spatial_scale=7.0, gs_iter_step=10, sh_degree=1)
    with pytest.raises(ValueError, match="capacity"):
        GT.GsTrainer(S_, sp, c2w, _K(), imgs, capacity=n - 1, **kw)
    with pytest.raises(ValueError, match=r"\[T,H,W,3\]"):
        GT.GsTrainer(S_, sp, c2w, _K(), imgs[..., :2].contiguous(), capacity=n, **kw)
    with pytest.raises(ValueError, match="poses"):
        GT.GsTrainer(S_, sp, c2w[:5], _K(), imgs, capacity=n, **kw)
    with pytest.raises(ValueError, match="pinned"):
        GT.GsTrainer(S_, sp, c2w, _K(), imgs.cpu(), capacity=n, **kw)
    saved = S_._pack
    S_._pack = {k: v.cpu() for k, v in saved.items()}
    try:
        with pytest.raises(ValueError, match="on the device"):
            GT.GsTrainer(S_, sp, c2w, _K(), imgs, capacity=n, **kw)
    finally:
        S_._pack = saved
    from gssdf_b200 import render as RD
    with pytest.raises(ValueError, match="eikonal_mode 1"):
        RD.GsSdfStep(100, 4, W, H, _dev(), 10000, S_.cfg, n_ray_samples=64, mlp_mode=1, eikonal_mode=0, delta_dev=S_.std_dev)
    G = _gs_trainer(room, S_, (c2w, imgs), 10)
    with pytest.raises(ValueError, match="give both"):
        G.T.load(sp["anchors"], sp["offsets"], sp["quaternion"], sp["scaling"], sp["opacity"], sp["features_dc"], sp["features_rest"],
                 S_.table, S_.mlp, sdf_exp_avg=S_.exp_avg)


def test_end_to_end_on_the_box_room(room):
    """SdfTrainer (200 iterations) -> neural_gs_init -> GsTrainer (colour init + 2000 joint iterations, SH degree 1) at 160x120 over 60
    training views; PSNR over 12 held-out views and the mesh of the jointly trained SDF. Measured on an H100: see DESIGN 7o."""
    S_ = _sdf_trainer(room, 200, seed=5, outlier_remove=True)
    c2w = _poses(72, 9)
    imgs = _images(c2w)
    train, test = slice(0, 60), slice(60, 72)
    G = _gs_trainer(room, S_, (c2w[train].contiguous(), imgs[train].contiguous()), 2000, sh_degree=1, capacity_mult=32, outlier_remove=True,
                    refine_gs_struct_start_iter=1000, densify=dict(refine_start_iter=200, refine_every=100), sh_degree_interval=500)
    G.run()
    h = G.histories()
    st = G.state()
    vms = torch.linalg.inv(c2w[test].to(torch.float64)).to(torch.float32)
    renders = torch.stack([st["render"](vm) for vm in vms])
    full, _ = MT.eval_render(renders.clamp(0, 1), imgs[test], [f"{i}.png" for i in range(12)])
    v, f, _ = ME.meshing(room["tree"], st["net"], room["margin"][0], room["margin"][1], 0.025)
    gt = S.box_wall_points(0.01)
    mm = ME.eval_mesh(v, f, torch.from_numpy(gt).to(_dev()), mesh_sample_point=1_000_000, gt_bbx_mask_on=False)
    print(f"held-out {full}; mesh {mm}; N_live {h['n_live'][-1]}; events {len(h['densify_events'])}; loss first {h['loss'][:3]} last "
          f"{h['loss'][-3:]}; sample_std last {h['sample_std'][-1]}")
    # measured on an H100: PSNR 28.7 dB (SSIM 0.943), accuracy 0.42 cm, completeness 0.56 cm, F-score 99.7 % at 2 cm
    assert full["PSNR"] > 24.0
    assert mm["MAE_accuracy (cm)"] < 1.0 and mm["MAE_completeness (cm)"] < 1.0 and mm["F-score (%)"] > 97.0
