"""The three densification kernels through cabi, and the Densifier's events on a GsSdfTrainer, against the fp64 arbiter of
tests/densify_oracle.py on the flip-free scenes of tests/densify_scenes.py.

Bars: exact wherever the kernel copies or decides (flags, counts, visibilities, radii, every copied parameter, moment, anchor and state
float, and every float it must leave alone); within C_ULP * 2^-24 * scale of fp64 wherever it computes (grad2d, the split offsets and
scalings), with no bad-entry fraction. Each test prints its worst |err| / (2^-24 scale).

C_ULP = 1. The worst ratios these tests printed on one H100 80GB HBM3 at a 700 W power limit: update_state 0.57, remap split rows
0.496, the Densifier's events 0.475 (update_state on the trainer 0.336)."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import densify_oracle as A  # noqa: E402
import densify_scenes as S  # noqa: E402


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _np(t):
    return t.detach().cpu().numpy()


def _check(label, got, want, scale=0.0):
    """fails on any entry beyond the bar; returns the worst |err| / (2^-24 scale) over the entries with a scale."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape, (label, got.shape, want.shape)
    scale = np.broadcast_to(np.asarray(scale, np.float64), want.shape)
    bad = A.off_bar(got, want, scale)
    if bad.any():
        i = int(np.argmax(bad.reshape(-1)))
        pytest.fail(f"{label}: {int(bad.sum())} / {bad.size} entries off; first at {np.unravel_index(i, want.shape)}: got "
                    f"{got.reshape(-1)[i]!r} want {want.reshape(-1)[i]!r} bound {A.C_ULP * A.U * scale.reshape(-1)[i]:.3e}")
    with np.errstate(invalid="ignore"):
        r = np.where(scale > 0, np.abs(got - want) / (A.U * np.where(scale > 0, scale, 1.0)), 0.0)
    r = r[np.isfinite(r)]
    return float(r.max()) if r.size else 0.0


# ---- update_state ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,C,with_radii,clamp", [(1, 1, True, False), (1, 3, True, True), (257, 1, False, False), (257, 3, True, True),
                                                  (30001, 1, True, False), (30001, 3, False, False), (30001, 3, True, True)])
def test_update_state_two_calls(N, C, with_radii, clamp):
    """Two accumulating calls. clamp: counts->nnz exceeds the buffer capacity by 17 (the kernel reads min(nnz, cap) rows); otherwise
    the buffers run 33 rows past nnz with a NaN gradient, visibility 2 and radius 10^4 on row 0. Rows outside gaussian_ids and the 64
    state floats past N keep their values bit for bit."""
    from gssdf_b200 import cabi
    dev = _dev()
    W, H = 1200, 680
    inp = S.render_inputs(N, C, W, H, seed=N + 10 * C)
    n = len(inp["gid"])
    cap = max(n - 17, 1) if clamp else n + 33
    m = min(n, cap)
    gid = np.zeros(cap, np.int64)
    v = np.full((cap, 2), np.nan, np.float32)
    vis = np.full((cap, 1), 2.0, np.float32)
    rad = np.full((cap, 2), 10000, np.int32)
    gid[:m], v[:m], vis[:m, 0], rad[:m] = inp["gid"][:m], inp["v"][:m], inp["vis"][:m], inp["radii"][:m]
    rng = np.random.default_rng(N)
    st0 = dict(grad2d=rng.uniform(0, 1e-3, N + 64), count=rng.integers(0, 5, N + 64), vis=rng.uniform(0, 0.5, N + 64),
               radii=rng.uniform(0, 0.05, N + 64))
    st0 = {k: v_.astype(np.float32) for k, v_ in st0.items()}
    if not with_radii:
        st0["radii"] = None
    st = {k: (_t(v_, dev) if v_ is not None else None) for k, v_ in st0.items()}
    counts = cabi.new_counts(dev, nnz=n)
    args = (_t(gid, dev), _t(v, dev), _t(vis, dev), _t(rad, dev) if with_radii else None)
    for _ in range(2):
        cabi.densify_update_state(N, cap, counts, *args, W, H, C, st["grad2d"], st["count"], st["vis"], st["radii"])
    torch.cuda.synchronize()
    two = lambda a: np.concatenate([a[:m], a[:m]])
    want, scale = A.update_state(st0, two(inp["gid"]), two(inp["v"]), two(inp["vis"]), two(inp["radii"]), W, H, C)
    worst = 0.0
    for k in A.STATE_NAMES:
        if st[k] is None:
            continue
        worst = max(worst, _check(f"N={N} C={C} {k}", _np(st[k]), want[k], scale[k]))
    print(f"update_state N={N} C={C} radii={with_radii} clamp={clamp}: worst grad2d |err| / (2^-24 scale) = {worst:.3g}")


# ---- flags ----------------------------------------------------------------------------------------------------------------------------
FLAG_MODES = {"grow+scale2d": dict(grow=True, use2d=True, vis=True, radii=True), "grow": dict(grow=True, use2d=False, vis=True, radii=True),
              "prune-only": dict(grow=False, use2d=False, vis=True, radii=True), "no-vis": dict(grow=True, use2d=True, vis=False, radii=True),
              "no-radii": dict(grow=True, use2d=True, vis=True, radii=False)}


@pytest.mark.parametrize("N", S.NS)
def test_flags_bit_exact(N):
    from gssdf_b200 import cabi
    dev = _dev()
    sc = S.flag_scene(N, 1, seed=N + 3)
    rows, c = sc["rows"], S.CFG
    pad = lambda a: _t(np.concatenate([a, np.full((64,) + a.shape[1:], np.nan, np.float32)]), dev)
    t = dict(offsets=pad(rows[:, 0:3]), quats=pad(rows[:, 3:7]), scaling=pad(rows[:, 7:10]), opacity=pad(rows[:, 10]), grad2d=pad(sc["grad2d"]),
             count=pad(sc["count"]), vis=pad(sc["vis"]), radii=pad(sc["radii"]))
    seen = 0
    for name, md in FLAG_MODES.items():
        out = torch.full((N + 64,), 0xAB, dtype=torch.uint8, device=dev)
        cabi.densify_flags(N, t["offsets"], t["quats"], t["scaling"], t["opacity"], out, grad2d=t["grad2d"] if md["grow"] else None,
                           count=t["count"] if md["grow"] else None, vis=t["vis"] if md["vis"] else None,
                           radii_state=t["radii"] if md["radii"] else None, grow_grad2d=c["grow_grad2d"], grow_scale3d=c["grow_scale3d"],
                           grow_scale2d=c["grow_scale2d"], use_scale2d=md["use2d"], prune_opa=c["prune_opa"], prune_scale3d=c["prune_scale3d"])
        want, _ = A.flags(rows, sc["grad2d"] if md["grow"] else None, sc["count"] if md["grow"] else None, sc["vis"] if md["vis"] else None,
                          sc["radii"] if md["radii"] else None, c["grow_grad2d"], c["grow_scale3d"], c["grow_scale2d"], md["use2d"], c["prune_opa"],
                          c["prune_scale3d"])
        got = _np(out)
        assert (got[N:] == 0xAB).all(), f"{name}: flags written past N"
        bad = np.nonzero(got[:N] != want)[0]
        assert not len(bad), f"N={N} {name}: {len(bad)} flags differ, first row {bad[0]} ({sc['cls'][bad[0]]}): got {got[bad[0]]:#x} want {want[bad[0]]:#x}"
        seen |= int(np.bitwise_or.reduce(want)) if N else 0
    if N >= len(S.CLASSES):
        assert seen == 127


# ---- remap ----------------------------------------------------------------------------------------------------------------------------
# (K, N, stride_old, stride_new, n_new, n_state, anchors_new)
REMAP_CASES = [(1, 1, 1, 5, 4, 0, False), (1, 30001, 30050, 61000, 60002, 4, True), (4, 255, 255, 300, 300, 1, True),
               (4, 256, 400, 256, 256, 2, False), (16, 257, 300, 520, 514, 3, True), (16, 30001, 40000, 30500, 30500, 4, True),
               (25, 256, 256, 1024, 777, 2, True), (25, 30001, 30001, 30001, 29000, 1, False)]


def _remap_gpu(case, dev, anchors_new=True):
    from gssdf_b200 import cabi
    old = {k: _t(v, dev) for k, v in case["old"].items()}
    new = {k: _t(v, dev) for k, v in case["new"].items()}
    if not anchors_new:
        new["anchors"] = None
    so, sn = [_t(s, dev) for s in case["states_old"]], [_t(s, dev) for s in case["states_new"]]
    cabi.densify_remap(case["n_new"], case["K"], case["stride_old"], case["stride_new"], _t(case["src"], dev), _t(case["mode"], dev),
                       _t(case["randn_row"], dev), _t(case["randn"], dev), old, new, so, sn)
    torch.cuda.synchronize()
    return new, sn


@pytest.mark.parametrize("K,N,so,sn,n_new,n_state,anchors_new", REMAP_CASES)
def test_remap_strided(K, N, so, sn, n_new, n_state, anchors_new):
    dev = _dev()
    case = S.remap_case(S.flag_scene(N, K, seed=K * 100 + N), so, sn, n_new, n_state, seed=N + K)
    new, sn_t = _remap_gpu(case, dev, anchors_new)
    want, scale = A.remap(K, so, sn, n_new, case["src"], case["mode"], case["randn_row"], case["randn"], case["old"],
                          dict(case["new"], anchors=case["new"]["anchors"] if anchors_new else None), case["states_old"], case["states_new"])
    lbl = f"K={K} N={N} stride {so}->{sn} n_new={n_new}"
    worst = _check(lbl + " params", _np(new["params"]), want["params"], scale)
    for k in ("exp_avg", "exp_avg_sq"):
        _check(f"{lbl} {k}", _np(new[k]), want[k])
    if anchors_new:
        _check(lbl + " anchors", _np(new["anchors"]), want["anchors"].reshape(-1))
    for i, s in enumerate(sn_t):
        _check(f"{lbl} state {i}", _np(s), want["states"][i])
    print(f"remap {lbl}: worst split |err| / (2^-24 scale) = {worst:.3g} over {int((case['mode'] == 2).sum())} split rows")


def test_remap_errors():
    from gssdf_b200 import _lib
    dev = _dev()
    case = S.remap_case(S.flag_scene(255, 4, seed=1), 255, 300, 300, 1, seed=2)
    case["n_new"] = 301
    case["src"], case["mode"], case["randn_row"] = (np.r_[a, a[:1]] for a in (case["src"], case["mode"], case["randn_row"]))
    with pytest.raises(_lib.GssdfError) as e:
        _remap_gpu(case, dev)
    assert e.value.code == -4  # GSSDF_ENOMEM
    from gssdf_b200 import cabi
    case = S.remap_case(S.flag_scene(255, 4, seed=1), 255, 255, 200, 0, seed=2)
    old = {k: _t(v, dev) for k, v in case["old"].items()}
    with pytest.raises(ValueError, match="in-place"):
        cabi.densify_remap(200, 4, 255, 255, _t(case["src"], dev), _t(case["mode"], dev), _t(case["randn_row"], dev), _t(case["randn"], dev),
                           old, old)


# ---- the Densifier on a trainer -------------------------------------------------------------------------------------------------------
def _rows(T, buf, n):
    return A.unpack(_np(buf[:A.row_floats(T.R.K) * T.N_cap]), n, T.R.K, T.N_cap)


def _cmp(label, T, D, want):
    n = T.N_live
    assert n == len(want["P"]), (label, n, len(want["P"]))
    w = _check(label + " params", _rows(T, T.params, n), want["P"], want["S"])
    _check(label + " exp_avg", _rows(T, T.exp_avg, n), want["M"])
    _check(label + " exp_avg_sq", _rows(T, T.exp_avg_sq, n), want["V"])
    _check(label + " anchors", _np(T.anchors), want["anchors"].reshape(-1, 3))
    for k in A.STATE_NAMES:
        _check(f"{label} state {k}", _np(D.state[k][:n]), want["state"][k])
    return w


@pytest.mark.parametrize("deg", [0, 3])
def test_densifier_events_on_trainer(deg):
    """update_state twice, then grow_gs, prune_gs, prune_nan_gs, prune_invisible_gs and reset_opacity at iteration 3100: past
    reset_every (3000, so the big-splat rule is live) and before refine_scale2d_stop_iter (4000, so the scale-2D rule is live). Before
    the first event three Adam steps visit a third of the rows each: at SH degree 3 the SH row groups are lazy and the rows a step did
    not visit are stale, so the surgery must bring them current (flush_sh) before it copies them. The reference is dense Adam on a copy
    of the buffers followed by the arbiter's events."""
    from gssdf_b200 import cabi, densify, render
    dev = _dev()
    K, N, W, H = (deg + 1) ** 2, 3000, 160, 96
    sc = S.trainer_scene(N, K, W, H, seed=deg + 5)
    cfg = dict(n_levels=16, n_features=2, log2_hashmap_size=19, base_resolution=32, per_level_scale=2.0, hidden_dim=64, n_hidden=3)
    T = render.GsSdfTrainer(2 * N + 100, K, W, H, dev, 100000, cfg, n_ray_samples=256, sh_degree=deg)
    r = sc["rows"]
    T.load(_t(np.random.default_rng(1).normal(size=(N, 3)).astype(np.float32), dev), _t(r[:, 0:3], dev), _t(r[:, 3:7], dev), _t(r[:, 7:10], dev),
           _t(r[:, 10], dev), _t(r[:, 11:14].reshape(N, 1, 3), dev), _t(r[:, 14:].reshape(N, K - 1, 3), dev), torch.zeros(T.n_table, device=dev),
           torch.zeros(T.n_mlp, device=dev))
    assert T.lazy_sh == (deg > 0)
    g = torch.Generator(dev).manual_seed(7)
    t0 = T.t0
    T._exp_avg[:t0].normal_(generator=g)
    T._exp_avg_sq[:t0].uniform_(generator=g)
    P2, M2, V2 = T._params[:t0].clone(), T._exp_avg[:t0].clone(), T._exp_avg_sq[:t0].clone()
    R = T.R
    for step in range(3):  # SH gradients on the visited rows only, every other gradient dense
        ids = torch.arange(step, N, 3, device=dev)
        grad = torch.zeros(t0, device=dev)
        grad[:T.seg_off[4]].normal_(generator=g)
        grad[T.seg_off[4]:] = 0
        for i in (4, 5):
            o, w = T.seg_off[i], T.seg_w[i]
            if w:
                seg = grad[o:o + N * w].view(N, w)
                seg[ids] = torch.randn(len(ids), w, device=dev, generator=g)
        for i in range(6):  # nothing beyond the live rows
            grad[T.seg_off[i] + N * T.seg_w[i]:T.seg_off[i] + T.N_cap * T.seg_w[i]] = 0
        R.p["gaussian_ids"][:len(ids)] = ids
        R.counts[0] = len(ids)
        T.flat_grad[:t0] = grad
        T.adam_all()
        cabi.adam_step(P2, grad.clone(), M2, V2, [gr[:4] for gr in T.splat_groups], T.t_splat)
    if deg > 0:
        assert T._sh_stale
    inp = sc["inputs"]
    n = len(inp["gid"])
    R.counts[0] = n
    R.p["gaussian_ids"][:n] = _t(inp["gid"], dev)
    R.g["v_densify"][:n] = _t(inp["v"], dev)
    R.r["visibilities"][:n, 0] = _t(inp["vis"], dev)
    R.p["radii"][:n] = _t(inp["radii"], dev)
    D = densify.Densifier(T, num_train_data=50, sh_degree=deg, refine_scale2d_stop_iter=4000, generator=torch.Generator(dev).manual_seed(11))
    for _ in range(2):
        D.update_state()
    st0 = {k: np.zeros(N, np.float32) for k in A.STATE_NAMES}
    two = lambda a: np.concatenate([a, a])
    want, scale = A.update_state(st0, two(inp["gid"]), two(inp["v"]), two(inp["vis"]), two(inp["radii"]), W, H, 1)
    worst = dict(update=0.0, events=0.0)
    for k in A.STATE_NAMES:
        worst["update"] = max(worst["update"], _check(f"deg {deg} update_state {k}", _np(D.state[k][:N]), want[k], scale[k]))
    it = 3100
    ev_cfg = dict(grow_grad2d=D.grow_grad2d, grow_scale3d=D.grow_scale3d, grow_scale2d=D.grow_scale2d, prune_opa=D.prune_opa,
                  prune_scale3d=D.prune_scale3d, spatial_scale=1.0, scale2d_stop=D.scale2d_stop)
    snap = A.snapshot(_rows(T, P2, N), _rows(T, M2, N), _rows(T, V2, N), _np(T.anchors), {k: _np(D.state[k][:N]) for k in A.STATE_NAMES})
    seen = 0

    def flags_of(snap, grow):
        f, m = A.event_flags(snap, ev_cfg, it, grow)
        lo = min(float(v_.min()) for v_ in m.values()) if len(f) else np.inf
        assert lo > S.MARGIN / 10, f"a decision lies {lo:.2e} from its threshold"
        return f

    # grow: the same randn stream as the Densifier's generator
    f = flags_of(snap, True)
    seen |= int(np.bitwise_or.reduce(f))
    gen = torch.Generator(dev)
    gen.set_state(D.gen.get_state())
    ns_want = int(((f & A.SPLIT) != 0).sum())
    randn = _np(torch.randn(2, ns_want, 3, device=dev, generator=gen).reshape(-1, 3))
    snap, nd, ns = A.grow_gs(snap, f, randn)
    assert D.grow_gs(it) == (nd, ns) and nd > 50 and ns > 100, (nd, ns)
    if deg > 0:
        assert bool((T.sh_last == T.t_sh).all())
    worst["events"] = max(worst["events"], _cmp(f"deg {deg} grow_gs", T, D, snap))
    snap = A.prune_gs(snap, flags_of(snap, False), it, D.reset_every)
    assert D.prune_gs(it) > 0
    worst["events"] = max(worst["events"], _cmp(f"deg {deg} prune_gs", T, D, snap))
    f = flags_of(snap, False)
    seen |= int(np.bitwise_or.reduce(f))
    snap = A.prune_nan_gs(snap, f)
    assert D.prune_nan_gs(it) > 0
    worst["events"] = max(worst["events"], _cmp(f"deg {deg} prune_nan_gs", T, D, snap))
    snap = A.prune_invisible_gs(snap, flags_of(snap, False), it, D.num_train_data)
    assert D.prune_invisible_gs(it) > 0
    worst["events"] = max(worst["events"], _cmp(f"deg {deg} prune_invisible_gs", T, D, snap))
    snap = A.reset_opacity(snap, D.prune_opa)
    D.reset_opacity()
    worst["events"] = max(worst["events"], _cmp(f"deg {deg} reset_opacity", T, D, snap))
    assert seen == 127, bin(seen)
    print(f"Densifier deg {deg}: N_live {N} -> {T.N_live}; worst |err| / (2^-24 scale): update_state {worst['update']:.3g}, "
          f"events {worst['events']:.3g}")
