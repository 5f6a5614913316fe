"""fp64 arbiter of one call of sdf_point_loss (gs-sdf_b200/csrc/sdf_loss.cuh) as gssdf_sdf_loss and the fused train kernel make it,
numpy only.

What it computes, per live point i < nl = min(n, n_live) (the reference: include/optimizer/loss.cpp:7-11,49-83, the softplus isigma of
include/neural_net/local_map.cpp:100-102, the sample gate and means of include/neural_mapping/neural_mapping.cpp:106-136,428-452):
  BCE       isigma = min(1 + softplus_100(y1) * bce_isigma, 500); z = -sdf * isigma; t = clamp(sigmoid(-gt * isigma), 1e-7f, 1 - 1e-7f);
            bce_weight * mean_i BCE-with-logits(z, t)
  coupling  0.5 * w * sdf^2, w = weight * gs_sdf_weight, times vis where vis > visible_thr and 0 elsewhere
  eikonal   V = 7: eikonal_weight * mean (|g| - 1)^2, g = the 6-offset central difference / (2 delta)
  gate      with n_gate (the coupling site): a point contributes to the coupling and eikonal terms only when (vis > visible_thr or no
            visibilities) and (valid_mask != 0 or no mask), and the eikonal mean divides by max(n_gate, 1) instead of nl. The BCE is the
            ray-sample site's term, which never runs gated; the gate does not touch it (as in the kernel).

Edge conventions are torch autograd's:
  - clamp_max(5e2) passes the gradient at equality (the kernel's `raw > 500` caps strictly);
  - clamp(lo, hi) passes it at both bounds;
  - the target is not detached: dL/dy1 carries the target's path -z w sigmoid'(-gt isigma) (-gt) where the clamp passes.
The clamp bounds are the fp32 scalars the reference clamps its fp32 tensor with: lo = 1e-7f, hi = 1 - 1e-7f = 1 - 2^-23. The reference's
target is the fp32 sigmoid 1 / (1 + exp(-x)), and just below 1 it has only the values 1 - 2^-23 and 1: it rises above hi only when
1 + exp(-x) rounds to 1, i.e. x >= 24 ln 2 (16.64), not where the exact sigmoid crosses hi (x = 15.94). Between the two the fp32 target
equals hi, the clamp does not engage and its gradient passes. This arbiter takes the fp32 rule for that one decision (TZ_HI); the kernel
and the reference agree with it. oracle.sdf_losses clamps at the fp64 bounds instead and differs from both inside that band.

Every computed value comes with an error scale (class E): the sum of the |terms| it is made of times the fp32 steps the kernel carries
them over, in units of 2^-24, so a GPU value must lie within C_ULP * 2^-24 * scale of the fp64 value whatever order the float atomics
add in. Decisions have margins (relative distance of the decisive quantity from its threshold); scenes keep them above MARGIN so that
GPU decisions equal the fp64 ones."""
import numpy as np

F32 = np.float32
U = 2.0 ** -24
C_ULP = 2.0
MARGIN = 1e-4
LO = float(F32(1e-7))
HI = float(F32(1.0) - F32(1e-7))       # 1 - 2^-23
TZ_LO = float(np.log(LO / (1.0 - LO)))  # sigmoid(x) < lo  <=>  x < TZ_LO (the fp32 sigmoid is accurate to an ulp there)
TZ_HI = 24.0 * np.log(2.0)              # fp32 sigmoid(x) > hi  <=>  fl(1 + exp(-x)) == 1  <=>  exp(-x) <= 2^-24
TZ_HI64 = float(np.log(HI / (1.0 - HI)))  # the exact sigmoid's crossing of hi (15.94): from here to TZ_HI lies the band
SP_THR, ISG_CAP = 20.0, 500.0
EXP_ULP, LOG_ULP = 2.0, 1.0             # CUDA expf / log1pf maximum errors


class E:
    """fp64 value and its error scale s: the fp32 kernel's value is within 2^-24 * s of v (each rounding adds |v|)."""

    def __init__(self, v, s=0.0):
        self.v = np.asarray(v, np.float64)
        self.s = np.zeros_like(self.v) + np.asarray(s, np.float64)

    def __neg__(self):
        return E(-self.v, self.s)

    def __add__(self, o):
        o = _e(o)
        v = self.v + o.v
        return E(v, self.s + o.s + np.abs(v))

    def __sub__(self, o):
        return self + (-_e(o))

    def __mul__(self, o):
        o = _e(o)
        v = self.v * o.v
        return E(v, np.abs(self.v) * o.s + np.abs(o.v) * self.s + np.abs(v))

    def __truediv__(self, o):
        o = _e(o)
        v = self.v / o.v
        return E(v, (self.s + np.abs(v) * o.s) / np.abs(o.v) + np.abs(v))


def _e(x):
    return x if isinstance(x, E) else E(x)


def where(c, a, b):
    a, b = _e(a), _e(b)
    return E(np.where(c, a.v, b.v), np.where(c, a.s, b.s))


def exp(a):
    v = np.exp(a.v)
    return E(v, v * (a.s + EXP_ULP))


def log1p(a):
    v = np.log1p(a.v)
    return E(v, a.s / (1.0 + a.v) + LOG_ULP * np.abs(v))


def sqrt(a):
    v = np.sqrt(a.v)
    with np.errstate(divide="ignore", invalid="ignore"):
        s = np.where(v > 0, a.s / (2 * np.where(v > 0, v, 1.0)) + v, np.sqrt(a.s))
    return E(v, s)


def sigmoid(a):
    return E(1.0) / (E(1.0) + exp(-a))


def _margin(x, t):
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.abs(np.asarray(x, np.float64) - t) / abs(t)


def f32(x):
    return float(F32(x))


def sdf_loss(sdf, y1, n, V, gt=None, weights=None, visibilities=None, visible_thr=0.0, valid_mask=None, gated=False, n_live=None,
             bce_isigma=10.0, bce_weight=1.0, eikonal_weight=0.1, gs_sdf_weight=1e-3, delta=0.1):
    """One call of sdf_point_loss over rows i < nl = min(n, n_live) of a layout of stride n (evaluation v*n + i is variant v of point i).
    sdf, y1: [V n] fp32; gt / weights / visibilities: [n] fp32 or None; valid_mask: [n] or None; gated: the caller passes n_gate (its
    value is the number of live rows that pass the gate, returned as n_gate). Scalars are rounded to fp32, as the args struct holds them.

    Returns a dict: loss (fp64) with loss_terms (sum of the per-point error scales) and loss_abs (sum of |per-point loss|), so that the
    bar of a sum added in `steps` fp32 additions is loss_scale(R, steps); v_sdf, v_y1 [V n] fp64 with NaN at rows >= nl (the kernel
    leaves them untouched) and their error scales; n_gate; dec: decision -> bool [nl]; margin: decision -> [nl] (inf where the decision
    does not apply); nl."""
    isig, bw, ew, gw, dl, thr = (f32(x) for x in (bce_isigma, bce_weight, eikonal_weight, gs_sdf_weight, delta, visible_thr))
    nl = n if n_live is None else max(min(int(n_live), n), 0)
    S = np.asarray(sdf, np.float32).astype(np.float64).reshape(V, n)[:, :nl]
    Y = np.asarray(y1, np.float32).astype(np.float64).reshape(V, n)[0, :nl] if y1 is not None else np.zeros(nl)
    inf = np.full(nl, np.inf)
    dec, margin = {}, {}
    ok = np.ones(nl, bool)
    if gated:
        if visibilities is not None:
            ok &= np.asarray(visibilities, np.float32)[:nl].astype(np.float64) > thr
        if valid_mask is not None:
            ok &= np.asarray(valid_mask)[:nl] != 0
    n_gate = int(ok.sum())
    dec["gate"] = ok
    s0 = E(S[0])
    part = E(np.zeros(nl))
    vs0 = E(np.zeros(nl))
    vy = E(np.zeros(nl))
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        if gt is not None:
            g = np.asarray(gt, np.float32).astype(np.float64)[:nl]
            by = E(Y) * 100.0
            lin = by.v > SP_THR
            L = log1p(exp(by))
            sp_log = E(L.v / 100.0, L.s / 100.0 + 1.5 * np.abs(L.v / 100.0))  # * 0.01f: its representation error and one rounding
            sp = where(lin, E(Y), sp_log)
            raw = E(1.0) + sp * isig
            capped = raw.v > ISG_CAP
            isg = where(capped, E(ISG_CAP), raw)
            tz = (-E(g)) * isg
            z = (-s0) * isg
            tsig = sigmoid(tz)
            tcl_lo, tcl_hi = tz.v < TZ_LO, tz.v >= TZ_HI
            tcl = tcl_lo | tcl_hi
            t = where(tcl_lo, E(LO), where(tcl_hi, E(HI), E(np.minimum(tsig.v, HI), tsig.s)))
            A = where(z.v > 0, z, E(0.0))
            bce = (A - z * t) + log1p(exp(-E(np.abs(z.v), z.s)))
            w = E(bw) / E(float(nl))
            part = part + w * bce
            dz = (sigmoid(z) - t) * w
            dt = (-z) * w
            vs0 = vs0 + dz * (-isg)
            gterm = dt * (tsig * (E(1.0) - tsig)) * (-g)
            d_isg = dz * (-s0) + where(tcl, E(0.0), gterm)
            vy = where(capped, E(0.0), (d_isg * isig) * where(lin, E(1.0), sigmoid(by)))
            dec.update(softplus_linear=lin, capped=capped, target_lo=tcl_lo, target_hi=tcl_hi, target_band=(tz.v > TZ_HI64) & ~tcl_hi)
            margin.update(softplus=_margin(by.v, SP_THR), cap=_margin(raw.v, ISG_CAP), target_lo=_margin(tz.v, TZ_LO),
                          target_hi=_margin(tz.v, TZ_HI))
        if weights is not None:
            w = E(np.asarray(weights, np.float32).astype(np.float64)[:nl]) * gw
            if visibilities is not None:
                vis = np.asarray(visibilities, np.float32).astype(np.float64)[:nl]
                vp = vis > thr
                w = where(vp, w * E(vis), E(0.0))
                dec["vis"] = vp
                margin["vis"] = _margin(vis, thr) if thr != 0 else np.where(vis == 0, 0.0, np.inf)
            if gated:
                w = where(ok, w, E(0.0))
            part = part + ((w * 0.5) * s0) * s0
            vs0 = vs0 + w * s0
        vs = [vs0] + [E(np.zeros(nl)) for _ in range(V - 1)]
        if V == 7:
            inv2d = E(0.5) / E(dl)
            gx, gy, gz = ((E(S[1 + 2 * k]) - E(S[2 + 2 * k])) * inv2d for k in range(3))
            nrm = sqrt((gx * gx + gy * gy) + gz * gz)
            we = E(ew) / E(float(max(n_gate, 1)) if gated else float(nl))
            we = where(gated & ~ok, E(0.0), we)
            part = part + we * ((nrm - 1.0) * (nrm - 1.0))
            z0 = nrm.v > 0
            k = where(z0, (((nrm - 1.0) * 2.0) / where(z0, nrm, E(1.0))) * we * inv2d, E(0.0))
            for j, gj in enumerate((gx, gy, gz)):
                vs[1 + 2 * j] = k * gj
                vs[2 + 2 * j] = -(k * gj)
            dec["norm_zero"] = ~z0
            # |g| = 0 only where every pair is bitwise equal, which any precision decides alike: no margin
    for key in ("softplus", "cap", "target_lo", "target_hi", "vis", "norm_zero"):
        margin.setdefault(key, inf)
    v_sdf, v_sdf_s = np.full((V, n), np.nan), np.zeros((V, n))
    v_y1, v_y1_s = np.full((V, n), np.nan), np.zeros((V, n))
    for v in range(V):
        v_sdf[v, :nl], v_sdf_s[v, :nl] = vs[v].v, vs[v].s
        v_y1[v, :nl] = vy.v if v == 0 else 0.0
        v_y1_s[v, :nl] = vy.s if v == 0 else 0.0
    return dict(loss=float(part.v.sum()), loss_terms=float(part.s.sum()), loss_abs=float(np.abs(part.v).sum()), part=part.v,
                v_sdf=v_sdf.reshape(-1), v_sdf_scale=v_sdf_s.reshape(-1), v_y1=v_y1.reshape(-1), v_y1_scale=v_y1_s.reshape(-1),
                n_gate=n_gate, dec=dec, margin=margin, nl=nl)


def loss_scale(R, steps, prefill=0.0):
    """error scale of loss_out = prefill + the per-point losses summed in `steps` fp32 additions (any order)"""
    return R["loss_terms"] + (R["loss_abs"] + abs(prefill)) * steps


def kernel_sum_steps(n, nl):
    """fp32 additions on the way of one point's loss into loss_out in sdf_loss_kernel: a 5-level warp tree, 8 warp partials, then one
    atomicAdd per 256-row block in an unspecified order (at most one per block with a live row)"""
    return 5 + 8 + -(-max(nl, 1) // 256)


def off_bar(got, want, scale):
    """entries of `got` beyond the GPU bar C_ULP * 2^-24 * scale (equal values, including NaN with NaN, always pass)"""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    with np.errstate(invalid="ignore"):
        ok = (got == want) | (np.isnan(got) & np.isnan(want)) | (np.abs(got - want) <= C_ULP * U * np.asarray(scale))
    return ~ok


def worst_ratio(got, want, scale):
    """max |got - want| / (2^-24 * scale) over the entries (0 where both are equal)"""
    got, want, scale = (np.asarray(a, np.float64) for a in (got, want, scale))
    d = np.abs(got - want)
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.where(d == 0, 0.0, d / (U * scale))
    r = r[np.isfinite(want)]
    return float(r.max()) if r.size else 0.0
