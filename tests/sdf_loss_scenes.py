"""Seeded per-point populations for the SDF loss (tests/sdf_loss_oracle.py), one designed class per block of rows, at the bce_sigma of
the shipped configurations: 1.0 (colmap/*, fast_livo/*), 0.1 (oxford_spires, GsSdfStep's default) and 0.01 (replica), with
bce_isigma = 1 / bce_sigma and delta = bce_sigma as GsSdfStep sets them.

Every row carries every input (sdf of the seven variants, y1, gt, weight, visibility, valid flag), and each row belongs to one class of
each family, so that a case picks its terms by the pointers it passes:
  bce       softplus in its log branch and its linear branch; isigma uncapped just under the cap and capped; target clamped low,
            clamped high, in the band between the exact sigmoid's and the fp32 sigmoid's upper bound (unclamped), unclamped; logits
            saturated in both signs (|z| in the hundreds)
  coupling  vis below visible_thr, above it, exactly at it (fails the strict >), valid_mask 0
  eikonal   |g| = 0 (bitwise-equal pairs), < 1, > 1, large
gt stays within the sampler's +-truncated_dis (3 x leaf size) of the configurations with that bce_sigma. Decisions within MARGIN
(relative) of their thresholds are moved away from them, so the GPU decides every row as the fp64 arbiter does."""
import numpy as np

import sdf_loss_oracle as SL

F32 = np.float32
ISIGMAS = (1.0, 10.0, 100.0)
# +-truncated_dis = 3 x leaf_sizes of the configurations that train each bce_sigma (replica 0.05; colmap / fast_livo / oxford up to 0.4)
TRUNC = {1.0: 1.2, 10.0: 1.2, 100.0: 0.15}
VISIBLE_THR = 0.1  # GsSdfStep's default
BCE_CLASSES = ("sp_log", "sp_linear", "uncapped_high", "capped", "target_lo", "target_hi", "target_band", "unclamped", "saturated_pos",
               "saturated_neg")
COUPLING_CLASSES = ("vis_below", "vis_above", "vis_at_thr", "invalid")
EIKONAL_CLASSES = ("norm_zero", "norm_lt1", "norm_gt1", "norm_large")
N_DEFAULT = 2347  # not a multiple of 256: the last block of sdf_loss_kernel is partial


def _sp_inv(sp):
    """y with softplus_100(y) = sp (sp > 0)"""
    return np.where(sp * 100 > 20, sp, np.log(np.expm1(np.minimum(sp * 100, 700))) / 100)


def _isg(y, isig):
    sp = np.where(100 * y > 20, y, np.log1p(np.exp(np.minimum(100 * y, 700))) / 100)
    return np.minimum(1 + sp * isig, 500.0)


def scene(isig, seed=0, n=N_DEFAULT):
    """dict(isig, sigma, delta, thr, sdf [7, n], y1 [7, n] (rows 1..6 NaN: the kernel reads variant 0 only), gt, w, vis, valid [n],
    classes: name -> bool [n]) in float32 / uint8"""
    rng = np.random.default_rng(int(seed * 1000 + isig))
    sigma = float(F32(1.0) / F32(isig))
    delta, thr, trunc = sigma, VISIBLE_THR, TRUNC[isig]
    u = lambda a, b, m: rng.uniform(a, b, m)
    cls = {}
    # ---- bce family: one block of rows per class, in a shuffled order
    bce_of = rng.permutation(np.arange(n) % len(BCE_CLASSES))
    y = np.zeros(n)
    gt = np.zeros(n)
    s0 = np.zeros(n)
    y_cap = lambda m: _sp_inv(u(1.05, 1.5, m) * 499.0 / isig)                   # raw in (525, 750)
    y_high = lambda m: _sp_inv(u(250.0, 490.0, m) / isig - 1.0 / isig)          # raw in (250, 490)
    for k, name in enumerate(BCE_CLASSES):
        m_ = bce_of == k
        cls[name] = m_
        m = int(m_.sum())
        if name == "sp_log":
            y[m_], gt[m_], s0[m_] = u(-0.5, 0.18, m), u(-trunc, trunc, m), u(-0.3, 0.3, m)
        elif name == "sp_linear":
            y[m_], gt[m_], s0[m_] = u(0.22, 3.0, m), u(-trunc, trunc, m), u(-0.3, 0.3, m)
        elif name == "uncapped_high":
            y[m_], gt[m_], s0[m_] = y_high(m), u(-trunc, trunc, m) * 0.02, u(-0.05, 0.05, m)
        elif name == "capped":
            y[m_], gt[m_], s0[m_] = y_cap(m), u(-trunc, trunc, m), u(-0.05, 0.05, m)
        elif name in ("target_lo", "target_hi", "target_band", "unclamped"):
            yy = np.where(rng.uniform(size=m) < 0.5, y_cap(m), y_high(m))
            isg = _isg(yy, isig)
            tz = {"target_lo": -u(16.5, 30.0, m), "target_hi": u(17.0, 30.0, m), "target_band": u(16.0, 16.6, m),
                  "unclamped": u(-15.5, 15.5, m)}[name]
            y[m_], gt[m_], s0[m_] = yy, -tz / isg, u(-0.05, 0.05, m)
        else:  # saturated logits z = -s0 isigma, |z| in [100, 550]
            yy = y_cap(m)
            z = u(100.0, 550.0, m) * (1 if name == "saturated_pos" else -1)
            y[m_], gt[m_], s0[m_] = yy, u(-trunc, trunc, m), -z / 500.0
    gt = np.clip(gt, -trunc, trunc)
    # ---- coupling family
    c_of = rng.permutation(np.arange(n) % len(COUPLING_CLASSES))
    w = u(0.05, 1.0, n)
    vis = np.zeros(n)
    valid = np.ones(n, np.uint8)
    for k, name in enumerate(COUPLING_CLASSES):
        m_ = c_of == k
        cls[name] = m_
        m = int(m_.sum())
        vis[m_] = {"vis_below": u(0.0, 0.98 * thr, m), "vis_above": u(1.02 * thr, 1.0, m), "vis_at_thr": np.full(m, float(F32(thr))),
                   "invalid": u(1.02 * thr, 1.0, m)}[name]
        if name == "invalid":
            valid[m_] = 0
    # ---- eikonal family: s[+k] - s[-k] = 2 delta g_k around a centre near s0
    e_of = rng.permutation(np.arange(n) % len(EIKONAL_CLASSES))
    d = rng.standard_normal((n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    nrm = np.zeros(n)
    for k, name in enumerate(EIKONAL_CLASSES):
        m_ = e_of == k
        cls[name] = m_
        m = int(m_.sum())
        nrm[m_] = {"norm_zero": np.zeros(m), "norm_lt1": u(0.2, 0.9, m), "norm_gt1": u(1.1, 3.0, m), "norm_large": u(50.0, 500.0, m)}[name]
    g = d * nrm[:, None]
    c = s0[:, None] + u(-0.02, 0.02, (n, 3))
    sdf = np.empty((7, n), F32)
    sdf[0] = s0
    for k in range(3):
        sdf[1 + 2 * k] = c[:, k] + g[:, k] * delta
        sdf[2 + 2 * k] = np.where(cls["norm_zero"], sdf[1 + 2 * k], c[:, k] - g[:, k] * delta)
    S = dict(isig=float(isig), sigma=sigma, delta=delta, thr=thr, trunc=trunc, sdf=sdf, gt=gt.astype(F32), w=w.astype(F32),
             vis=vis.astype(F32), valid=valid, classes=cls)
    S["y1"] = np.full((7, n), np.nan, F32)
    S["y1"][0] = y
    _nudge(S)
    return S


def arbiter(S, V=7, gt=True, w=True, vis=True, gated=False, n_live=None, **kw):
    """sdf_loss_oracle.sdf_loss on the scene with the chosen inputs and the GsSdfStep weights (bce 1, eikonal 0.1, gs_sdf 1e-3)"""
    n = S["sdf"].shape[1]
    return SL.sdf_loss(S["sdf"][:V].reshape(-1), S["y1"][:V].reshape(-1), n, V, gt=S["gt"] if gt else None, weights=S["w"] if w else None,
                       visibilities=S["vis"] if vis else None, visible_thr=S["thr"], valid_mask=S["valid"] if gated else None,
                       gated=gated, n_live=n_live, bce_isigma=S["isig"], bce_weight=kw.get("bce_weight", 1.0),
                       eikonal_weight=kw.get("eikonal_weight", 0.1), gs_sdf_weight=kw.get("gs_sdf_weight", 1e-3), delta=S["delta"])


def near(R):
    """rows with some decision within MARGIN of its threshold (vis exactly at the threshold is exact in any precision: not counted)"""
    m = R["margin"]
    return (m["softplus"] < SL.MARGIN) | (m["cap"] < SL.MARGIN) | (m["target_lo"] < SL.MARGIN) | (m["target_hi"] < SL.MARGIN) | (
        (m["vis"] < SL.MARGIN) & (m["vis"] > 0))


def _nudge(S, rounds=8):
    for _ in range(rounds):
        bad = near(arbiter(S))
        if not bad.any():
            return
        y, gt, vis = S["y1"][0], S["gt"], S["vis"]
        y[bad] = (y[bad].astype(np.float64) * (1 + 3e-3) + 1e-4).astype(F32)
        gt[bad] = (gt[bad].astype(np.float64) * (1 - 3e-3)).astype(F32)
        vis[bad & ~S["classes"]["vis_at_thr"]] *= F32(1 + 3e-3)
    raise AssertionError("sdf_loss_scenes: could not move every decision off its threshold")
