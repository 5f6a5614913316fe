"""fp64 composition of gssdf_sdf_train in its analytic-eikonal mode (eikonal_mode 1), built from the oracle chains of oracle/oracle.py
(TEST INFRASTRUCTURE ONLY).

What the fused kernel computes, per live base point i (rows < n_live), in the arrangement of the training step:
  coordinates   x01 = fl(fl((x - origin) * inv_size) + 0.5) in float32 (load_x); the six variants add +-delta to one world coordinate
                first, in float32
  first order   BCE on (sdf, y1) (mean over n_live) + gs_sdf 0.5 w s^2 with w = weight * gs_sdf_weight, times vis where vis > thr and 0
                elsewhere, and 0 for a point the gate rejects -> dL/dsdf, dL/dy1 -> table / decoder gradient and dL/dx (x01 units, scaled
                by inv_size into world units)
  second order  g = g01 * inv_size (g01 = the analytic gradient in x01 units), gnum from the variants with delta in world units;
                eikonal_weight * mean (|g| - 1)^2 + align_weight * mean |g - gnum| over the gated points (over n_gate when a gate is
                given, else over n_live) -> c = dL/dg, handed back as c * inv_size = dL/dg01 -> double backward to table and decoder
The second-order part does not reach dL/dx.

Knife edges: the comparison with an fp32 / tensor-core kernel is only meaningful where fp32-grade differences cannot flip a discrete
choice, so the input builders keep only points whose smallest |hidden pre-activation| is at least 1e-4 (a ReLU that may switch) and
whose analytic and numerical gradients differ by at least 2e-3 |g| in every component (the sign in the align loss)."""
import numpy as np

f32 = np.float32
OFFSETS = np.array([[0, 0, 0], [1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.float32)
HIDDEN = 64
PREACT_EDGE = 1e-4
ALIGN_EDGE = 2e-3
HALF_Q, HALF_MIN_NORMAL = 2.0 ** -24, 2.0 ** -14  # fp16 subnormal quantum, smallest normal
HALF_EDGE = 3e-5


def make_mlp(rng, n_hidden, in_dim=32, hidden=HIDDEN):
    dims = [in_dim] + [hidden] * (1 + n_hidden) + [2]
    ps = []
    for k, o in zip(dims[:-1], dims[1:]):
        b = 1 / np.sqrt(k)
        ps += [rng.uniform(-b, b, o * k), rng.uniform(-b, b, o)]
    return np.concatenate(ps).astype(np.float32)


def world_to_x01(xw, origin, inv_size):
    """load_x: fl(fl((x - origin) * inv_size) + 0.5), two float32 roundings (no fused multiply-add); inv_size 0 = x is already in x01."""
    xw = np.asarray(xw, f32)
    if not inv_size:
        return xw.copy()
    d = (xw - np.asarray(origin, f32).reshape(1, 3)).astype(f32)
    return ((d * f32(inv_size)).astype(f32) + f32(0.5)).astype(f32)


def variant_world(xw, delta):
    """[6, n, 3]: variants 1..6 (+x, -x, +y, -y, +z, -z), the offset added in world units in float32"""
    xw = np.asarray(xw, f32)
    return (xw[None] + OFFSETS[1:, None] * f32(delta)).astype(f32)


def min_preact(O, x01, table, mlp, n_hidden):
    """smallest |hidden pre-activation| of each point (fp64 decoder on the oracle's features)"""
    feat = O.hashgrid_fwd(x01, table)
    a, o, K = feat.astype(np.float64), 0, feat.shape[1]
    m = np.full(len(feat), np.inf)
    for _ in range(1 + n_hidden):
        W = mlp[o:o + HIDDEN * K].reshape(HIDDEN, K).astype(np.float64)
        b = mlp[o + HIDDEN * K:o + HIDDEN * K + HIDDEN].astype(np.float64)
        o += HIDDEN * K + HIDDEN
        z = a @ W.T + b
        m = np.minimum(m, np.abs(z).min(1))
        a, K = np.maximum(z, 0), HIDDEN
    return m


def point_terms(O, xw, table, mlp, n_hidden, origin, inv_size, delta, variants=True):
    """Per-point oracle quantities (independent across points, so any subset may be taken by indexing)."""
    x01 = world_to_x01(xw, origin, inv_size)
    sdf, y1, _ = O.sdf_fwd(x01, table, mlp, HIDDEN, n_hidden)
    g01 = O.sdf_grad_analytic(x01, table, mlp, HIDDEN, n_hidden).astype(np.float64)
    P = dict(xw=np.asarray(xw, f32), x01=x01, sdf=np.asarray(sdf, np.float64), y1=np.asarray(y1, np.float64), g01=g01,
             pre=min_preact(O, x01, table, mlp, n_hidden), gnum=None)
    if variants:
        xv = world_to_x01(variant_world(xw, delta).reshape(-1, 3), origin, inv_size)
        s = np.asarray(O.sdf_fwd(xv, table, mlp, HIDDEN, n_hidden)[0], np.float64).reshape(6, -1)
        P["gnum"] = np.stack([s[0] - s[1], s[2] - s[3], s[4] - s[5]], 1) * (0.5 / delta)  # delta in world units: gnum in world units
    return P


def half_edges(dfeat, rel=HALF_EDGE):
    """Rows whose first-order feature cotangent dL/dy has a subnormal element within rel x (the row's largest |dL/dy|) of an fp16
    rounding midpoint. tcnn's binding rounds dL/dy to fp16 before its x128 loss scale; with means over tens of thousands of points these
    cotangents are fp16 subnormals (quantum 6e-8, about a tenth of a typical value), so an fp32-grade difference that moves one across a
    midpoint changes that row's dL/dx by a whole quantum. Their dL/dx is left out of the comparison; their gradients stay in."""
    a = np.abs(np.asarray(dfeat, np.float64))
    dist = np.abs(np.mod(a / HALF_Q, 1.0) - 0.5) * HALF_Q
    return ((a < HALF_MIN_NORMAL) & (dist < rel * a.max(1, keepdims=True))).any(1)


def take(P, idx):
    return {k: (None if v is None else v[idx]) for k, v in P.items()}


def knife_edges(P, inv_size):
    isz = inv_size or 1.0
    edge = P["pre"] < PREACT_EDGE
    if P["gnum"] is not None:
        g = P["g01"] * isz
        edge |= (np.abs(g - P["gnum"]) < ALIGN_EDGE * np.linalg.norm(g, axis=1, keepdims=True)).any(1)
    return edge


def clean_points(O, rng, n_keep, table, mlp, n_hidden, origin, inv_size, delta, half_extent, variants=True):
    """n_keep world points in the cube origin +- half_extent, none on a knife edge, with their point terms. Candidates are drawn 2.5x,
    screened by the cheap pre-activation test, and the full terms are computed for just over n_keep survivors."""
    if n_keep == 0:
        return point_terms(O, np.zeros((0, 3), f32), table, mlp, n_hidden, origin, inv_size, delta, variants)
    cand = (np.asarray(origin, f32) + rng.uniform(-half_extent, half_extent, (int(2.5 * n_keep) + 64, 3))).astype(f32)
    pre = min_preact(O, world_to_x01(cand, origin, inv_size), table, mlp, n_hidden)
    cand = cand[pre >= PREACT_EDGE][:int(1.1 * n_keep) + 64]
    P = point_terms(O, cand, table, mlp, n_hidden, origin, inv_size, delta, variants)
    keep = np.flatnonzero(~knife_edges(P, inv_size))
    assert len(keep) >= n_keep, f"only {len(keep)} of {n_keep} candidates off the knife edges"
    return take(P, keep[:n_keep])


# ------------------------------------------------------------------------------------------------------------------------------
# the composition's glue: pure functions of per-point values, pinned against torch.autograd by the host test
# ------------------------------------------------------------------------------------------------------------------------------
def gate(n_live, visibilities=None, valid_mask=None, visible_thr=0.0, gated=False):
    """(ok [n_live] bool, divisor of the second-order means). With a gate (n_gate given to the kernel) a point passes when vis > thr and
    valid_mask != 0 and the means divide by the number that pass (at least 1); without one every live point counts and the means divide
    by n_live."""
    if not gated:
        return np.ones(n_live, bool), max(n_live, 1)
    ok = np.ones(n_live, bool)
    if visibilities is not None:
        ok &= np.asarray(visibilities, np.float32)[:n_live] > f32(visible_thr)
    if valid_mask is not None:
        ok &= np.asarray(valid_mask)[:n_live] != 0
    return ok, max(int(ok.sum()), 1)


def coupling_weights(weights, gs_sdf_weight, visibilities, visible_thr, ok):
    """per-point factor w of the gs_sdf term 0.5 w s^2: weight * gs_sdf_weight, times vis where vis > thr (0 elsewhere), 0 where the
    gate rejects the point"""
    w = np.asarray(weights, np.float64) * gs_sdf_weight
    if visibilities is not None:
        vis = np.asarray(visibilities, np.float32)[:len(w)]
        w = np.where(vis > f32(visible_thr), w * vis.astype(np.float64), 0.0)
    return np.where(ok, w, 0.0)


def second_order_terms(g01, gnum, inv_size, eikonal_weight, align_weight, ok, nl):
    """loss and its cotangent dL/dg01 [n, 3] of eikonal + align on the analytic gradient: g = g01 * inv_size (world units), means over
    nl, rows outside `ok` contribute nothing; the cotangent goes back into x01 units as c * inv_size."""
    isz = inv_size or 1.0
    g = np.asarray(g01, np.float64) * isz
    okf = np.asarray(ok, np.float64)[:, None]
    nrm = np.linalg.norm(g, axis=1)
    we = eikonal_weight / nl
    loss = we * float((okf[:, 0] * (nrm - 1) ** 2).sum())
    c = we * np.where(nrm > 0, 2 * (nrm - 1) / np.where(nrm > 0, nrm, 1), 0)[:, None] * g
    if gnum is not None and align_weight > 0:
        d = g - gnum
        wa = align_weight / (3 * nl)
        loss += wa * float((okf * np.abs(d)).sum())
        c = c + wa * np.sign(d)
    return loss, c * okf * isz


def compose(O, P, table, mlp, n_hidden, inv_size, delta, eikonal_weight, align_weight, n_live, gt=None, bce_isigma=10.0, bce_weight=0.0,
            weights=None, gs_sdf_weight=0.0, visibilities=None, valid_mask=None, visible_thr=0.0, gated=False):
    """gssdf_sdf_train(eikonal_mode 1) on the live points P (rows 0 .. n_live-1). Returns dict(loss, loss1, loss2, mlp (total), table1,
    mlp1, table2, mlp2 (first- / second-order shares), v_x [n_live, 3] world units, n_gate). The table total is left to the caller
    (table1 + table2): at 15 M parameters one fp64 copy fewer per case matters."""
    isz = inv_size or 1.0
    assert len(P["sdf"]) == n_live
    ok, nl2 = gate(n_live, visibilities, valid_mask, visible_thr, gated)
    w_eff = None if weights is None else coupling_weights(weights, gs_sdf_weight, visibilities, visible_thr, ok)
    loss1, v_s, v_y = O.sdf_losses(P["sdf"], P["y1"], n_live, 1, gt_sdf=gt, weights=w_eff, bce_isigma=bce_isigma, bce_weight=bce_weight,
                                   eikonal_weight=0.0, gs_sdf_weight=1.0, delta=delta)
    tg1, mg1, dx = O.sdf_bwd(P["x01"], table, mlp, v_s, v_y, HIDDEN, n_hidden)
    dfeat, _ = O.mlp_bwd(O.hashgrid_fwd(P["x01"], table), [32] + [HIDDEN] * (1 + n_hidden) + [2], mlp, np.stack([v_s, v_y], 1))
    loss2, c01 = second_order_terms(P["g01"], P["gnum"], inv_size, eikonal_weight, align_weight, ok, nl2)
    sel = np.flatnonzero(ok)
    tg2, mg2 = O.sdf_grad_analytic_bwd(P["x01"][sel], table, mlp, c01[sel].astype(np.float32), HIDDEN, n_hidden)
    R = dict(loss=loss1 + loss2, loss1=loss1, loss2=loss2, mlp=mg1 + mg2, table1=tg1, mlp1=mg1, table2=tg2, mlp2=mg2,
             v_x=np.asarray(dx, np.float64) * isz, n_gate=int(ok.sum()))
    R["v_x_edge"] = half_edges(dfeat)
    for k, v in R.items():
        assert np.all(np.isfinite(v)), f"oracle {k} is not finite: keep the table amplitudes small (fp16 x128 intermediates)"
    return R


def add(*Rs):
    """sum of compositions that accumulate into the same buffers (stage [A] then stage [C])"""
    return {k: sum(R[k] for R in Rs) for k in ("loss", "mlp", "table1", "mlp1", "table2", "mlp2")}
