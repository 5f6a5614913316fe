"""Seeded densification scenes (numpy only), flip-free by construction.

A scene is a population of splat rows, one designed class per row, with the statistics the flag kernel reads:

  plain        low gradient, mid-size, opaque, visible: no flag
  dupli        high gradient, max(sx, sy) <= grow_scale3d                      -> DUPLI
  split_grad   high gradient, max(sx, sy) > grow_scale3d                       -> SPLIT
  split_2d     low gradient, radii > grow_scale2d                              -> SPLIT while use_scale2d, else nothing
  split_prune  split_grad with opacity < prune_opa                             -> SPLIT | P_OPA
  nan_j        a NaN in column j of offsets | quaternion | scaling (j < 10)    -> P_NAN
  invisible    vis < 1e-4 (some exactly 0)                                     -> P_INVIS
  small        min(sx, sy) < 1e-4                                              -> P_SMALL
  big          max(sx, sy) > prune_scale3d                                     -> P_BIG

Quaternion norms span 1e-3 to 1e3, some have w ~ 0 and one is all zero; scales span 1e-5 to 1. After drawing, `nudge` moves any row
whose fp64 decision lies within MARGIN (relative) of its threshold away from it until none does, so the GPU's fp32 decisions equal the
fp64 ones bit for bit. Non-small classes keep min(sx, sy) >= 3e-4 and non-big ones max(sx, sy) <= 0.08, so a split child's
log(s / 1.6) clears the prune thresholds as well."""
import numpy as np

import densify_oracle as A

MARGIN = 1e-4
CLASSES = ("plain", "dupli", "split_grad", "split_2d", "split_prune", "invisible", "small", "big") + tuple(f"nan_{j}" for j in range(10))
# Densifier defaults (config/base.yaml), spatial scale 1
CFG = dict(grow_grad2d=2e-4, grow_scale3d=0.01, grow_scale2d=0.05, prune_opa=0.05, prune_scale3d=0.1, spatial_scale=1.0)
KS = (1, 4, 16, 25)
NS = (1, 255, 256, 257, 30001)


def _logu(rng, lo, hi, n):
    return np.exp(rng.uniform(np.log(lo), np.log(hi), n))


def classes(N, rng):
    """every class once before any repeats (N >= len(CLASSES)), in a shuffled order"""
    return np.array(CLASSES)[rng.permutation(N) % len(CLASSES)]


def draw_rows(cls, K, rng):
    """fp32 row matrix [N, 11 + 3K] for the classes `cls`."""
    N = len(cls)
    rows = np.zeros((N, A.row_floats(K)), np.float64)
    rows[:, 0:3] = rng.normal(0, 0.01, (N, 3))
    d = rng.normal(size=(N, 4))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    q = d * _logu(rng, 1e-3, 1e3, N)[:, None]
    wz = rng.random(N) < 0.15
    q[wz, 0] = rng.normal(0, 1e-7, wz.sum()) * np.abs(q[wz, 1])  # w ~ 0
    if N > 1:
        q[rng.integers(N)] = 0.0
    rows[:, 3:7] = q
    s = _logu(rng, 3e-4, 8e-3, (N, 2))
    big_s = np.isin(cls, ("split_grad", "split_prune"))
    s[big_s] = _logu(rng, 1.2e-2, 8e-2, (big_s.sum(), 2))
    ax = rng.integers(0, 2, N)
    sm, bg = cls == "small", cls == "big"
    s[sm, ax[sm]] = _logu(rng, 1e-5, 8e-5, sm.sum())
    s[bg, ax[bg]] = _logu(rng, 0.12, 1.0, bg.sum())
    rows[:, 7:9] = np.log(s)
    rows[:, 9] = np.log(_logu(rng, 1e-5, 1.0, N))
    o = rng.uniform(0.06, 0.99, N)
    lo = cls == "split_prune"
    o[lo] = rng.uniform(0.005, 0.045, lo.sum())
    rows[:, 10] = np.log(o / (1 - o))
    rows[:, 11:] = rng.normal(0, 0.5, (N, 3 * K))
    for j in range(10):
        rows[cls == f"nan_{j}", j] = np.nan
    return rows.astype(np.float32)


def draw_stats(cls, rng):
    """designed per-row gradient (per count), count, vis and radii_state"""
    N = len(cls)
    high = np.isin(cls, ("dupli", "split_grad", "split_prune"))
    g = _logu(rng, 1e-6, 1.5e-4, N)
    g[high] = _logu(rng, 3e-4, 1e-2, high.sum())
    count = rng.integers(0, 9, N).astype(np.float64)
    count[high] = np.maximum(count[high], 1)
    vis = rng.uniform(1e-3, 1.0, N)
    inv = cls == "invisible"
    vis[inv] = np.where(rng.random(inv.sum()) < 0.3, 0.0, _logu(rng, 1e-7, 8e-5, inv.sum()))
    radii = rng.uniform(0.0, 0.04, N)
    radii[rng.random(N) < 0.1] = 0.0
    r2 = cls == "split_2d"
    radii[r2] = rng.uniform(0.06, 0.5, r2.sum())
    return g, count, vis, radii


def nudge_once(rows, grad2d, count, vis, radii, cfg=CFG, grad_rows=None):
    """One pass over the decisions of `A.flags` (grow on, use_scale2d on, vis on): every one within MARGIN of its threshold is moved
    away from it, in place. grad2d (or the callback grad_rows(i, factor) for update_state inputs), radii and vis scale by 1 -+ 1e-3,
    the deciding log-scale or the opacity logit steps by 1e-3. Returns True when nothing had to move."""
    f, m = A.flags(rows, grad2d, count, vis, radii, cfg["grow_grad2d"], cfg["grow_scale3d"], cfg["grow_scale2d"], True, cfg["prune_opa"],
                   cfg["prune_scale3d"])
    bad = {k: np.nonzero(v < MARGIN)[0] for k, v in m.items()}
    if not any(len(b) for b in bad.values()):
        return True
    sx, sy = np.exp(rows[:, 7].astype(np.float64)), np.exp(rows[:, 8].astype(np.float64))
    away = lambda x, t: np.where(x > np.float32(t), 1.0, -1.0)
    i = bad["grad"]
    if len(i):
        fac = 1 + 1e-3 * away(grad2d[i] / np.maximum(count[i], 1), cfg["grow_grad2d"])
        if grad_rows is None:
            grad2d[i] = (grad2d[i] * fac).astype(np.float32)
        else:
            grad_rows(i, fac)
    for rule, t, pick in (("scale3d", cfg["grow_scale3d"], np.fmax), ("big", cfg["prune_scale3d"], np.fmax), ("small", 1e-4, np.fmin)):
        i = bad[rule]
        if len(i):
            v = pick(sx[i], sy[i])
            rows[i, np.where(v == sx[i], 7, 8)] += (1e-3 * away(v, t)).astype(np.float32)
    i = bad["opacity"]
    if len(i):
        rows[i, 10] += (1e-3 * away(1 / (1 + np.exp(-rows[i, 10].astype(np.float64))), cfg["prune_opa"])).astype(np.float32)
    for k, arr, t in (("scale2d", radii, cfg["grow_scale2d"]), ("vis", vis, 1e-4)):
        i = bad[k]
        if len(i):
            arr[i] = (arr[i] * (1 + 1e-3 * away(arr[i], t))).astype(arr.dtype)
    return False


def nudge(rows, grad2d, count, vis, radii, cfg=CFG, max_iter=60):
    for _ in range(max_iter):
        if nudge_once(rows, grad2d, count, vis, radii, cfg):
            return
    raise AssertionError("nudge did not converge")


def flag_scene(N, K, seed):
    """rows + fp32 statistics, nudged; cls per row."""
    rng = np.random.default_rng(seed)
    cls = classes(N, rng)
    rows = draw_rows(cls, K, rng)
    g, count, vis, radii = draw_stats(cls, rng)
    grad2d = (g * np.maximum(count, 1)).astype(np.float32)
    count, vis, radii = count.astype(np.float32), vis.astype(np.float32), radii.astype(np.float32)
    nudge(rows, grad2d, count, vis, radii)
    return dict(N=N, K=K, cls=cls, rows=rows, grad2d=grad2d, count=count, vis=vis, radii=radii)


def render_inputs(N, C, W, H, seed, nnz_per_cam=None):
    """update_state inputs of C cameras: each camera sees a random sorted subset of the N splats, so a splat seen by several cameras
    appears once per camera in gaussian_ids. v_densify spans 1e-9..1e-3, radii [0, 400] with zeros, visibilities [0, 1] with zeros."""
    rng = np.random.default_rng(seed)
    per = nnz_per_cam or max(1, (2 * N) // 3)
    gid = np.concatenate([np.sort(rng.choice(N, min(per, N), replace=False)) for _ in range(C)]).astype(np.int64)
    n = len(gid)
    v = rng.normal(size=(n, 2)) * _logu(rng, 1e-9, 1e-3, n)[:, None]
    v[rng.random(n) < 0.05] = 0.0
    vis = rng.uniform(0, 1, n)
    vis[rng.random(n) < 0.1] = 0.0
    radii = rng.integers(0, 400, (n, 2))
    radii[rng.random(n) < 0.1] = 0
    return dict(gid=gid, v=v.astype(np.float32), vis=vis.astype(np.float32), radii=radii.astype(np.int32), W=W, H=H, C=C)


def trainer_scene(N, K, W, H, seed):
    """rows for GsSdfTrainer.load and one camera's update_state inputs, meant to be applied twice: every splat but the invisible ones
    with zero visibility appears once, so the state then holds count 2, grad = the designed gradient and the designed vis and radii.
    radii are integers and cannot be nudged: r / max(W, H) must miss grow_scale2d by the choice of W and H (checked)."""
    rng = np.random.default_rng(seed)
    cls = classes(N, rng)
    rows = draw_rows(cls, K, rng)
    g, _, vis, radii = draw_stats(cls, rng)
    gid = np.nonzero(vis > 0)[0].astype(np.int64)
    th = rng.uniform(0, 2 * np.pi, len(gid))
    v = np.stack([g[gid] * np.cos(th) / (W * 0.5), g[gid] * np.sin(th) / (H * 0.5)], 1).astype(np.float32)
    r = np.round(radii[gid] * max(W, H)).astype(np.int32)
    rr = np.stack([r, rng.integers(0, np.maximum(r, 1)).astype(np.int32)], 1)
    flip = rng.random(len(gid)) < 0.5
    rr[flip] = rr[flip][:, ::-1]
    inp = dict(gid=gid, v=v, vis=vis[gid].astype(np.float32), radii=rr, W=W, H=H, C=1)
    pos = np.full(N, -1)
    pos[gid] = np.arange(len(gid))

    def grad_rows(i, fac):
        j = pos[i]
        inp["v"][j[j >= 0]] = (inp["v"][j[j >= 0]] * fac[j >= 0][:, None]).astype(np.float32)

    for _ in range(60):
        st = {k: np.zeros(N, np.float32) for k in A.STATE_NAMES}
        for _ in range(2):
            o, _s = A.update_state(st, inp["gid"], inp["v"], inp["vis"], inp["radii"], W, H, 1)
            st = {k: o[k].astype(np.float32) for k in A.STATE_NAMES}
        vis_in, radii_in = st["vis"].copy(), st["radii"].copy()
        if nudge_once(rows, st["grad2d"].copy(), st["count"], vis_in, radii_in, grad_rows=grad_rows):
            return dict(N=N, K=K, cls=cls, rows=rows, inputs=inp)
        assert np.array_equal(radii_in, st["radii"]), "a radius lies on the grow_scale2d threshold"
        inp["vis"] = vis_in[gid]
    raise AssertionError("trainer scene did not clear its margins")


SENTINEL = np.float32(-1.5e38)  # what the new buffers hold before a remap: every float the kernel must not write keeps it


def remap_case(sc, stride_old, stride_new, n_new, n_state, seed, dens_order=False):
    """densify_remap inputs over a flag scene's rows: old flat buffers of row capacity stride_old (NaN beyond the N rows), moments
    N(0, 1) and U(0, 1), anchors, n_state state arrays; src rows with repeats in arbitrary order and modes 0 / 1 / 2 mixed (at least
    one of each when n_new >= 3); randn rows for the split samples. New buffers of capacity stride_new hold SENTINEL."""
    rng = np.random.default_rng(seed)
    N, K = sc["N"], sc["K"]
    rf = A.row_floats(K)
    nan = np.full(rf * stride_old, np.nan, np.float32)
    old = dict(params=A.pack(sc["rows"], K, stride_old, nan),
               exp_avg=A.pack(rng.normal(size=(N, rf)).astype(np.float32), K, stride_old, nan),
               exp_avg_sq=A.pack(rng.uniform(size=(N, rf)).astype(np.float32), K, stride_old, nan),
               anchors=np.r_[rng.normal(size=(N, 3)), np.full((stride_old - N, 3), np.nan)].astype(np.float32).reshape(-1))
    src = rng.integers(0, N, n_new).astype(np.int32)
    mode = rng.integers(0, 3, n_new).astype(np.uint8)
    mode[:min(3, n_new)] = np.arange(min(3, n_new))
    n_split = int((mode == 2).sum())
    randn = rng.normal(size=(max(n_split, 1) + 5, 3)).astype(np.float32)
    randn_row = np.where(mode == 2, rng.permutation(len(randn))[:n_new] if n_new <= len(randn) else rng.integers(0, len(randn), n_new), 0)
    new = {k: np.full(rf * stride_new, SENTINEL, np.float32) for k in ("params", "exp_avg", "exp_avg_sq")}
    new["anchors"] = np.full(3 * stride_new, SENTINEL, np.float32)
    states_old = [np.r_[rng.uniform(size=N), np.full(stride_old - N, np.nan)].astype(np.float32) for _ in range(n_state)]
    states_new = [np.full(stride_new, SENTINEL, np.float32) for _ in range(n_state)]
    return dict(K=K, stride_old=stride_old, stride_new=stride_new, n_new=n_new, src=src, mode=mode, randn_row=randn_row.astype(np.int32),
                randn=randn, old=old, new=new, states_old=states_old, states_new=states_new)
