"""fp64 arbiter of the densification kernels (gs-sdf_b200/csrc/densify.cu) and of the Densifier events built on them
(gssdf_b200/densify.py), numpy only.

A splat row is the kernel's row of 11 + 3K floats: columns 0-2 offsets, 3-6 quaternion, 7-9 scaling (log), 10 opacity (logit), 11-13
features_dc, 14.. features_rest. In the flat buffers segment s starts at (its first column) * stride and row r of a segment of width w
sits at r * w; `segments` is that column -> (segment start, width, index) map.

Every computed value comes with an error scale: the sum of the |terms| it is made of times the fp32 steps the kernel carries them over,
so that a GPU value must lie within C_ULP * 2^-24 * scale of the fp64 value whatever order the atomics add in. Copies and decisions have
no scale: they must be exact.

`mut` names one-line mistakes a kernel could make (MUTATIONS); tests/test_densify_host.py checks that each of them moves some output of
the scenes beyond the GPU bar, so the GPU tests would catch it."""
import numpy as np

DUPLI, SPLIT, P_OPA, P_SMALL, P_BIG, P_NAN, P_INVIS = 1, 2, 4, 8, 16, 32, 64
FLAG_NAMES = {DUPLI: "dupli", SPLIT: "split", P_OPA: "opacity", P_SMALL: "small", P_BIG: "big", P_NAN: "nan", P_INVIS: "invisible"}
U = 2.0 ** -24
F32 = np.float32
STATE_NAMES = ("grad2d", "count", "vis", "radii")
C_ULP = 1.0
MUTATIONS = (("swap_R01",), ("one_s",), ("no_1.6",), ("no_ncam",), ("swap_WH",), ("dc_rest",), ("K3=3K",), ("no_scale2d",),
             ("keep_dup_moments",)) + tuple((f"nan_col_{j}",) for j in range(10))
# fp32 steps of one update_state term |(v0 W/2 C, v1 H/2 C)|: two products per component, the squares and their sum, the square root
TERM_STEPS = 4
# split offsets, fp32 steps per |term|: v + R(q^) (s^2 randn)_xy. q^ = q / max(|q|, 1e-12) carries ~3 roundings per component, so an
# entry of R (at most 2 in size) is off by <= 16 ulp absolute; e = s s randn with s = expf (2 ulp) is off by <= 6 ulp relative; the
# product and the two-term sum add ~4 more. The offset itself goes through two roundings.
SPLIT_E_STEPS, SPLIT_OFF_STEPS = 26, 2
SPLIT_F = float(F32(1.6))  # the kernel and the reference divide by the float 1.6f


def off_bar(got, want, scale=0.0):
    """entries of `got` beyond the GPU bar: not equal to `want` (NaN matches NaN, inf matches inf) and more than C_ULP * 2^-24 * scale
    away from it (scale 0: the entry must be exact)."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    with np.errstate(invalid="ignore"):
        same = (got == want) | (np.isnan(got) & np.isnan(want)) | (np.abs(got - want) <= C_ULP * U * np.asarray(scale))
    return ~same


def row_floats(K):
    return 11 + 3 * K


def segments(K, mut=()):
    """[11 + 3K] (pre, w, k) of every column c, as densify_remap_kernel maps it."""
    K3 = 3 * K if "K3=3K" in mut else 3 * (K - 1)
    dc_end = 13 if "dc_rest" in mut else 14
    c = np.arange(row_floats(K))
    conds = [c < 3, c < 7, c < 10, c < 11, c < dc_end]
    pre = np.select(conds, [0, 3, 7, 10, 11], 14)
    w = np.select(conds, [3, 4, 3, 1, 3], K3)
    return pre, w, c - pre


def flat_index(rows, K, stride, mut=()):
    """[len(rows), 11 + 3K] positions of the rows' columns in a flat buffer of row capacity `stride`."""
    pre, w, k = segments(K, mut)
    return pre[None] * np.int64(stride) + np.asarray(rows, np.int64)[:, None] * w[None] + k[None]


def pack(rows, K, stride, base=None):
    """row matrix [n, 11 + 3K] -> flat buffer [(11 + 3K) * stride] (`base` supplies everything the rows do not cover)."""
    rows = np.asarray(rows)
    out = np.zeros(row_floats(K) * stride, rows.dtype) if base is None else np.array(base, rows.dtype)
    out[flat_index(np.arange(len(rows)), K, stride)] = rows
    return out


def unpack(flat, n, K, stride):
    return np.asarray(flat)[flat_index(np.arange(n), K, stride)]


def _take(a, idx):
    return np.asarray(a)[np.clip(idx, 0, len(a) - 1)]  # a mutated map may point outside a buffer; the clip only matters there


# ---- update_state -------------------------------------------------------------------------------------------------------------------
def update_state(state0, gaussian_ids, v_densify, visibilities, radii, W, H, n_cameras, mut=()):
    """NeuralGS::update_state on the state arrays `state0` (dict of fp32 [N]; state0["radii"] None when radii are not tracked) for the
    nnz rows given (the caller clamps nnz to the buffer capacity). Returns (expected fp64 dict, error-scale dict): grad2d += the fp64
    norms, count += 1 per row, vis = max(vis, visibility), radii = max(radii, fl32(max(rx, ry) / max(W, H))) -- the fp32 division is
    correctly rounded, so count, vis and radii are exact."""
    N = len(state0["grad2d"])
    gid = np.asarray(gaussian_ids, np.int64)
    v = np.asarray(v_densify, np.float64)
    fw, fh = (H, W) if "swap_WH" in mut else (W, H)
    c = 1 if "no_ncam" in mut else n_cameras
    t = np.hypot(v[:, 0] * fw * 0.5 * c, v[:, 1] * fh * 0.5 * c)
    n = np.bincount(gid, minlength=N)
    g0 = np.asarray(state0["grad2d"], np.float64)
    tsum = np.bincount(gid, t, minlength=N)
    out = dict(grad2d=g0 + tsum, count=np.asarray(state0["count"], np.float64) + n)
    vis = np.array(state0["vis"], np.float64)
    np.maximum.at(vis, gid, np.maximum(np.asarray(visibilities, np.float64), 0.0))
    out["vis"] = vis
    scale = dict(grad2d=(np.abs(g0) + tsum) * (TERM_STEPS + n), count=np.zeros(N), vis=np.zeros(N))
    if state0.get("radii") is not None and radii is not None:
        r = np.asarray(radii)
        q = np.maximum(r[:, 0], r[:, 1]).astype(F32) / F32(max(W, H))
        rad = np.array(state0["radii"], np.float64)
        np.maximum.at(rad, gid, np.maximum(q.astype(np.float64), 0.0))
        out["radii"], scale["radii"] = rad, np.zeros(N)
    return out, scale


# ---- flags --------------------------------------------------------------------------------------------------------------------------
def _margin(x, t):
    """relative distance of x from the threshold t (inf where x is NaN: a NaN decides the same way in any precision)."""
    with np.errstate(invalid="ignore", divide="ignore"):
        m = np.abs(x - t) / abs(t)
    return np.where(np.isnan(m), np.inf, m)


def flags(rows, grad2d=None, count=None, vis=None, radii=None, grow_grad2d=0.0, grow_scale3d=0.0, grow_scale2d=0.0, use_scale2d=False,
          prune_opa=0.0, prune_scale3d=np.inf, mut=()):
    """densify_flags_kernel in fp64 on the row matrix (columns 0-10 are read). Thresholds are rounded to fp32 as the args struct holds
    them. Returns (flags uint8 [N], margins: rule -> [N] relative distance of the decisive quantity from its threshold).

    The kernel's fmaxf / fminf over (sx, sy) return the other axis when one is NaN (np.fmax / np.fmin here), where torch's max of the
    reference propagates the NaN; the Densifier prunes NaN rows before every grow and prune, so no event sees the difference."""
    rows = np.asarray(rows, np.float64)
    N = len(rows)
    g2, g3, gs2, popa, pbig = (float(F32(x)) for x in (grow_grad2d, grow_scale3d, grow_scale2d, prune_opa, prune_scale3d))
    small_t, vis_t = float(F32(1e-4)), float(F32(1e-4))
    with np.errstate(over="ignore", invalid="ignore"):
        sx, sy = np.exp(rows[:, 7]), np.exp(rows[:, 8])
        smax, smin = np.fmax(sx, sy), np.fmin(sx, sy)
        opa = 1.0 / (1.0 + np.exp(-rows[:, 10]))
    f = np.zeros(N, np.uint8)
    inf = np.full(N, np.inf)
    m = dict(grad=inf, scale3d=inf, scale2d=inf, opacity=_margin(opa, popa), small=_margin(smin, small_t), big=_margin(smax, pbig),
             vis=inf)
    if grad2d is not None and count is not None:
        grad = np.asarray(grad2d, np.float64) / np.maximum(np.asarray(count, np.float64), 1.0)
        high, small = grad > g2, smax <= g3
        f |= np.where(high & small, DUPLI, 0).astype(np.uint8)
        split = high & ~small
        if (use_scale2d or "no_scale2d" in mut) and radii is not None:
            r = np.asarray(radii, np.float64)
            split |= r > gs2
            m["scale2d"] = _margin(r, gs2)
        f |= np.where(split, SPLIT, 0).astype(np.uint8)
        m["grad"], m["scale3d"] = _margin(grad, g2), _margin(smax, g3)
    f |= np.where(opa < popa, P_OPA, 0).astype(np.uint8)
    f |= np.where(smin < small_t, P_SMALL, 0).astype(np.uint8)
    f |= np.where(smax > pbig, P_BIG, 0).astype(np.uint8)
    cols = [j for j in range(10) if f"nan_col_{j}" not in mut]
    f |= np.where(np.isnan(rows[:, cols]).any(1), P_NAN, 0).astype(np.uint8)
    if vis is not None:
        v = np.asarray(vis, np.float64)
        f |= np.where(v < vis_t, P_INVIS, 0).astype(np.uint8)
        m["vis"] = _margin(v, vis_t)
    return f, m


# ---- remap --------------------------------------------------------------------------------------------------------------------------
def split_sample(q, scaling, offsets, rn, mut=()):
    """offsets + R(q / max(|q|, 1e-12)) (s*s*randn) with s = (exp(scaling.xy), 0), and its error scale; all [n, 3] fp64."""
    q = np.asarray(q, np.float64)
    q = q / np.maximum(np.sqrt((q * q).sum(1)), 1e-12)[:, None]
    w, x, y, z = q.T
    c0 = np.stack([1 - 2 * (y * y + z * z), 2 * (x * y + w * z), 2 * (x * z - w * y)], 1)  # columns 0 and 1 of the rotation matrix
    c1 = np.stack([2 * (x * y - w * z), 1 - 2 * (x * x + z * z), 2 * (y * z + w * x)], 1)
    if "swap_R01" in mut:
        c0, c1 = c1, c0
    s = np.exp(np.asarray(scaling, np.float64)[:, :2])
    e = (s if "one_s" in mut else s * s) * np.asarray(rn, np.float64)[:, :2]
    off = np.asarray(offsets, np.float64)
    out = off + c0 * e[:, :1] + c1 * e[:, 1:2]
    scale = SPLIT_OFF_STEPS * np.abs(off) + SPLIT_E_STEPS * (np.abs(e[:, :1]) + np.abs(e[:, 1:2]))
    return out, scale


def split_scaling(scaling, mut=()):
    """log(exp(scaling.xy) / 1.6f), and -inf for z; error scale 4 + 2 |result| (expf 2 ulp relative, the division, logf 1 ulp)."""
    s = np.asarray(scaling, np.float64)
    xy = s[:, :2] - (0.0 if "no_1.6" in mut else np.log(SPLIT_F))
    out = np.concatenate([xy, np.full((len(s), 1), -np.inf)], 1)
    scale = np.concatenate([4 + 2 * np.abs(xy), np.zeros((len(s), 1))], 1)
    return out, scale


def remap(K, stride_old, stride_new, n_new, src, mode, randn_row, randn, old, new, states_old=(), states_new=(), mut=()):
    """densify_remap_kernel. old: dict(params, exp_avg, exp_avg_sq, anchors) of flat fp32 arrays; new: the same keys holding what the
    new buffers contain before the call (anchors may be None). Returns (expected dict of fp64 flat arrays incl. "states",
    params error scale): the new buffers with rows < n_new rewritten and every other float as it was."""
    src = np.asarray(src, np.int64)[:n_new]
    mode = np.asarray(mode)[:n_new]
    io = flat_index(src, K, stride_old, mut)
    inn = flat_index(np.arange(n_new), K, stride_new, mut)
    P = _take(old["params"], io).astype(np.float64)
    S = np.zeros_like(P)
    sp = np.nonzero(mode == 2)[0]
    if len(sp):
        s = src[sp]
        po = np.asarray(old["params"])
        q = po[3 * stride_old + s[:, None] * 4 + np.arange(4)]
        sc = po[7 * stride_old + s[:, None] * 3 + np.arange(3)]
        rn = np.asarray(randn).reshape(-1, 3)[np.asarray(randn_row)[sp]]
        P[sp, 0:3], S[sp, 0:3] = split_sample(q, sc, P[sp, 0:3], rn, mut)
        P[sp, 7:10], S[sp, 7:10] = split_scaling(P[sp, 7:10], mut)
    keep = (mode == 0) | ((mode == 1) if "keep_dup_moments" in mut else False)
    out = {}
    for name, val in (("params", P), ("exp_avg", None), ("exp_avg_sq", None)):
        if val is None:
            val = np.where(keep[:, None], _take(old[name], io), 0.0)
        buf = np.array(new[name], np.float64)
        buf[np.clip(inn, 0, len(buf) - 1)] = val
        out[name] = buf
    scale = np.zeros(len(out["params"]))
    scale[np.clip(inn, 0, len(scale) - 1)] = S
    if new.get("anchors") is not None:
        a = np.array(new["anchors"], np.float64).reshape(-1, 3)
        a[:n_new] = np.asarray(old["anchors"]).reshape(-1, 3)[src]
        out["anchors"] = a
    out["states"] = []
    for so, sn in zip(states_old, states_new):
        st = np.array(sn, np.float64)
        st[:n_new] = np.asarray(so)[src]
        out["states"].append(st)
    return out, scale


# ---- the Densifier's events on a snapshot -------------------------------------------------------------------------------------------
def snapshot(P, M, V, anchors, state, S=None):
    """A trainer's live rows: P, M, V row matrices [n, 11 + 3K] (params, exp_avg, exp_avg_sq), anchors [n, 3], state dict of [n] arrays,
    S the error scale of P (zeros: every value exact)."""
    P = np.asarray(P, np.float64)
    return dict(P=P, M=np.asarray(M, np.float64), V=np.asarray(V, np.float64), anchors=np.asarray(anchors, np.float64),
                state={k: np.asarray(state[k], np.float64) for k in STATE_NAMES}, S=np.zeros_like(P) if S is None else S)


def remap_rows(snap, src, mode, randn_row=None, randn=None, mut=()):
    """`remap` on a snapshot: the rows src[r] under mode[r]; error scales travel with copied rows."""
    n, rf = snap["P"].shape
    K = (rf - 11) // 3
    n_new = len(src)
    old = {k: pack(snap[s], K, n) for k, s in (("params", "P"), ("exp_avg", "M"), ("exp_avg_sq", "V"))}
    old["anchors"] = snap["anchors"].reshape(-1)
    new = {k: np.zeros(row_floats(K) * n_new) for k in ("params", "exp_avg", "exp_avg_sq")}
    new["anchors"] = np.zeros(3 * n_new)
    st = [snap["state"][k] for k in STATE_NAMES]
    o, sc = remap(K, n, n_new, n_new, src, mode, randn_row, randn, old, new, st, [np.zeros(n_new)] * 4, mut)
    S = unpack(sc, n_new, K, n_new)
    S = np.where(S > 0, S, snap["S"][np.asarray(src)])
    return dict(P=unpack(o["params"], n_new, K, n_new), M=unpack(o["exp_avg"], n_new, K, n_new), V=unpack(o["exp_avg_sq"], n_new, K, n_new),
                anchors=o["anchors"], state=dict(zip(STATE_NAMES, o["states"])), S=S)


def event_flags(snap, cfg, it, with_grow):
    """Densifier._flags: cfg holds the Densifier's thresholds (grow_grad2d, grow_scale3d, grow_scale2d, prune_opa, prune_scale3d, the
    spatial scales and scale2d_stop)."""
    st = snap["state"]
    return flags(snap["P"], st["grad2d"] if with_grow else None, st["count"] if with_grow else None, st["vis"], st["radii"],
                 cfg["grow_grad2d"], cfg["grow_scale3d"] * cfg["spatial_scale"], cfg["grow_scale2d"], it < cfg["scale2d_stop"],
                 cfg["prune_opa"], cfg["prune_scale3d"] * cfg["spatial_scale"])


def grow_gs(snap, f, randn):
    """Densifier.grow_gs with flags f: rows [non-split rows in order | duplicates | split k=0 | split k=1]; randn [2 n_split, 3] in the
    order of torch.randn(2, n_split, 3). Returns (snapshot, n_dupli, n_split)."""
    n = len(f)
    di = np.nonzero(f & DUPLI)[0]
    is_split = np.r_[(f & SPLIT) != 0, np.zeros(len(di), bool)]
    src1, mode1 = np.r_[np.arange(n), di], np.r_[np.zeros(n, np.uint8), np.ones(len(di), np.uint8)]
    sel, rest = np.nonzero(is_split)[0], np.nonzero(~is_split)[0]
    ns = len(sel)
    if not (len(di) or ns):
        return snap, 0, 0
    src = np.r_[src1[rest], src1[sel], src1[sel]]
    mode = np.r_[mode1[rest], np.full(2 * ns, 2, np.uint8)]
    randn_row = np.r_[np.zeros(len(rest), np.int64), np.arange(2 * ns)]
    return remap_rows(snap, src, mode, randn_row, randn), len(di), ns


def prune(snap, is_prune):
    if not is_prune.any():
        return snap
    valid = np.nonzero(~is_prune)[0]
    return remap_rows(snap, valid, np.zeros(len(valid), np.uint8))


def prune_gs(snap, f, it, reset_every, prune_opa_only=False):
    m = P_OPA | P_SMALL | (P_BIG if (not prune_opa_only and it > reset_every) else 0)
    return prune(snap, (f & m) != 0)


def prune_nan_gs(snap, f):
    return prune(snap, (f & P_NAN) != 0)


def prune_invisible_gs(snap, f, it, num_train_data):
    if not (it > 0 and it % num_train_data == 0):
        return snap
    snap = dict(snap, state=dict(snap["state"], vis=np.zeros_like(snap["state"]["vis"])))
    return prune(snap, (f & P_INVIS) != 0)


def reset_opacity(snap, prune_opa):
    """opacity = min(opacity, logit(2 prune_opa)) (the fp32 clamp bound the Densifier passes), opacity moments zeroed."""
    cap = float(F32(np.log(2 * prune_opa / (1 - 2 * prune_opa))))
    out = {k: np.array(v) for k, v in snap.items() if k != "state"}
    out["state"] = snap["state"]
    out["P"][:, 10] = np.minimum(out["P"][:, 10], cap)
    out["M"][:, 10] = 0.0
    out["V"][:, 10] = 0.0
    return out
