"""The SDF loss arbiter (tests/sdf_loss_oracle.py) and its scenes (tests/sdf_loss_scenes.py) on the CPU:
  - the arbiter equals float64 torch autograd of the reference's expressions (loss.cpp sdf_loss / eikonal_loss / gs_sdf_loss, the softplus
    isigma of local_map.cpp:100-102, the gate and means of neural_mapping.cpp:428-452), gated and ungated, with a live count;
  - without gate, visibilities or live count it equals oracle.sdf_losses, except for the rows whose target lies in the band where the
    fp32 sigmoid the reference clamps has not yet left 1 - 2^-23 (there only the target's gradient differs, by design);
  - every scene sets every class and keeps every decision off its threshold;
  - a float32 numpy transcription of sdf_loss.cuh meets the GPU bar on every scene and case, and each of its one-line mutations moves
    some output beyond the bar on some scene (so the GPU test would catch it)."""
import numpy as np
import pytest

import sdf_loss_oracle as SL
import sdf_loss_scenes as SC

F32 = np.float32
CASES = {  # name -> (V, gt, weights, vis, gated): the argument sets of the GPU test
    "v7_gt": (7, True, False, False, False),
    "v1_gt": (1, True, False, False, False),
    "v7_w": (7, False, True, False, False),
    "v7_w_vis": (7, False, True, True, False),
    "v7_w_vis_gate": (7, False, True, True, True),
    "v1_w_vis_gate": (1, False, True, True, True),
}
DEAD = 301  # rows at or past n_live
W32 = (float(F32(0.1)), float(F32(1e-3)))  # eikonal / gs_sdf weights as the args struct holds them


@pytest.fixture(scope="module", params=SC.ISIGMAS, ids=lambda s: f"isig{s:g}")
def scene(request):
    return SC.scene(request.param)


# ---- the arbiter against float64 autograd of the reference expressions -------------------------------------------------------------
def _torch_reference(S, V, gt, w, vis, gated, n_live, bce_w=1.0, eik_w=0.1, gs_w=1e-3):
    torch = pytest.importorskip("torch")
    Fn = torch.nn.functional
    n = S["sdf"].shape[1]
    nl = min(n_live, n)
    f = lambda a: float(F32(a))
    isig, thr, delta = f(S["isig"]), f(S["thr"]), f(S["delta"])
    sdf = torch.tensor(S["sdf"][:V, :nl].astype(np.float64), requires_grad=True)
    y1 = torch.tensor(S["y1"][0, :nl].astype(np.float64), requires_grad=True)
    loss = torch.zeros((), dtype=torch.float64)
    if gt:
        g = torch.tensor(S["gt"][:nl].astype(np.float64))
        isigma = (1 + Fn.softplus(y1, beta=100, threshold=20) * isig).clamp_max(5e2)  # local_map.cpp:100-102, loss.cpp:52
        tz = -g * isigma
        t = torch.sigmoid(tz).clamp(SL.LO, SL.HI)
        # the fp32 sigmoid stays at 1 - 2^-23 up to tz = 24 ln 2: there the clamp does not engage and its gradient passes
        band = (tz.detach() > np.log(SL.HI / (1 - SL.HI))) & (tz.detach() < SL.TZ_HI)
        ts = torch.sigmoid(tz)
        t = torch.where(band, ts + (SL.HI - ts).detach(), t)
        loss = loss + f(bce_w) * Fn.binary_cross_entropy_with_logits(-sdf[0] * isigma, t)
    ok = torch.ones(nl, dtype=torch.bool)
    if gated:
        ok = torch.tensor(S["vis"][:nl].astype(np.float64) > thr) & torch.tensor(S["valid"][:nl] != 0)
    if w:
        ww = torch.tensor(S["w"][:nl].astype(np.float64)) * f(gs_w)
        if vis:
            v = torch.tensor(S["vis"][:nl].astype(np.float64))
            ww = torch.where(v > thr, ww * v, torch.zeros_like(ww))
        sel = ok.nonzero().squeeze(1)
        loss = loss + 0.5 * (ww[sel] * sdf[0][sel].square()).sum()  # loss.cpp:7-11
    if V == 7:
        sel = ok.nonzero().squeeze(1)
        if len(sel):
            s = sdf[:, sel]
            grad = (0.5 / delta) * torch.stack([s[1] - s[2], s[3] - s[4], s[5] - s[6]], 1)  # local_map.cpp:127-131
            loss = loss + f(eik_w) * (grad.norm(2, 1) - 1.0).square().mean()  # loss.cpp:81-83
    loss.backward()
    gs = sdf.grad.numpy() if sdf.grad is not None else np.zeros((V, nl))
    gy = y1.grad.numpy() if y1.grad is not None else np.zeros(nl)
    return float(loss.detach()), gs, gy


@pytest.mark.parametrize("case", sorted(CASES))
def test_arbiter_matches_autograd_of_the_reference(scene, case):
    V, gt, w, vis, gated = CASES[case]
    n = scene["sdf"].shape[1]
    for n_live in (n, n - DEAD):
        R = SC.arbiter(scene, V, gt, w, vis, gated, n_live=n_live)
        loss, gs, gy = _torch_reference(scene, V, gt, w, vis, gated, n_live)
        nl = R["nl"]
        vs = R["v_sdf"].reshape(V, n)
        tol = 1e-4 * SL.U
        assert abs(R["loss"] - loss) <= tol * SL.loss_scale(R, 1), (case, R["loss"], loss)
        assert not SL.off_bar(vs[:, :nl] / 1e4, gs / 1e4, R["v_sdf_scale"].reshape(V, n)[:, :nl] * 1e-8).any(), case
        assert not SL.off_bar(R["v_y1"][:nl] / 1e4, gy / 1e4, R["v_y1_scale"][:nl] * 1e-8).any(), case
        assert np.isnan(vs[:, nl:]).all() and np.isnan(R["v_y1"].reshape(V, n)[:, nl:]).all()
        if gated:
            assert R["n_gate"] == int(((scene["vis"][:nl] > F32(scene["thr"])) & (scene["valid"][:nl] != 0)).sum())


def test_arbiter_matches_oracle_sdf_losses_off_the_band(scene, oracle):
    """no gate, visibilities or live count: oracle.sdf_losses, which clamps the target at the fp64 bounds. Off the band
    (15.94 < -gt isigma < 24 ln 2) it agrees to 1e-4 of the GPU bar on unclamped rows and within the bar on clamped ones."""
    n = scene["sdf"].shape[1]
    R = SC.arbiter(scene, 7, True, True, False, False)
    band = R["dec"]["target_band"]
    assert band[scene["classes"]["target_band"]].all()
    keep = ~band
    S2 = dict(scene, sdf=scene["sdf"][:, keep], y1=scene["y1"][:, keep], gt=scene["gt"][keep], w=scene["w"][keep], vis=scene["vis"][keep])
    R2 = SC.arbiter(S2, 7, True, True, False, False)
    m = int(keep.sum())
    lo, vs, vy = oracle.sdf_losses(S2["sdf"].reshape(-1), np.r_[S2["y1"][0], np.zeros(6 * m, F32)], m, 7,
                                   S2["gt"], S2["w"], S2["isig"], 1.0, *W32, S2["delta"])
    # oracle.sdf_losses clamps at 1e-7 and 1 - 1e-7, the fp32 reference at 1e-7f and 1 - 2^-23: on the clamped rows the targets differ
    # by 1.2e-15 and 1.9e-8, which stays inside the GPU bar; every other row agrees to 1e-4 of it
    clamped = np.tile(R2["dec"]["target_lo"] | R2["dec"]["target_hi"], 7)
    k = np.where(clamped, 1.0, 1e-4)
    assert abs(R2["loss"] - lo) <= 1e-2 * SL.U * SL.loss_scale(R2, 1)
    assert not SL.off_bar(R2["v_sdf"] / k, vs / k, R2["v_sdf_scale"]).any()
    assert not SL.off_bar(R2["v_y1"] / k, vy / k, R2["v_y1_scale"]).any()
    # inside the band the fp64 clamp drops the target's path of dL/dy1 from 16.12 on and the fp32 reference keeps it; that path is
    # dt sigmoid'(tz) gt with 1 - sigmoid ~ 1e-7, one fp32 step of 1, so either convention meets the GPU bar there
    _, _, vy_all = oracle.sdf_losses(scene["sdf"].reshape(-1), np.r_[scene["y1"][0], np.zeros(6 * n, F32)], n, 7, scene["gt"], scene["w"],
                                     scene["isig"], 1.0, *W32, scene["delta"])
    assert not SL.off_bar(R["v_y1"][:n], vy_all[:n], R["v_y1_scale"][:n]).any()


# ---- scenes ---------------------------------------------------------------------------------------------------------------------------
def test_scenes_set_every_class_and_clear_every_margin(scene):
    cls = scene["classes"]
    for name in SC.BCE_CLASSES + SC.COUPLING_CLASSES + SC.EIKONAL_CLASSES:
        assert cls[name].sum() >= 50, name
    R = SC.arbiter(scene)
    d = R["dec"]
    assert not SC.near(R).any()
    assert (scene["gt"] >= -scene["trunc"]).all() and (scene["gt"] <= scene["trunc"]).all()
    # each class reaches its branch
    assert not d["softplus_linear"][cls["sp_log"]].any() and d["softplus_linear"][cls["sp_linear"]].all()
    assert d["capped"][cls["capped"]].all() and not d["capped"][cls["uncapped_high"]].any()
    assert d["target_lo"][cls["target_lo"]].all() and d["target_hi"][cls["target_hi"]].all()
    for c in ("target_band", "unclamped"):
        assert not (d["target_lo"] | d["target_hi"])[cls[c]].any(), c
    tz_band = -scene["gt"][cls["target_band"]].astype(np.float64) * np.minimum(
        1 + np.where(100 * scene["y1"][0][cls["target_band"]] > 20, scene["y1"][0][cls["target_band"]], 0) * scene["isig"], 500)
    assert (tz_band > np.log(SL.HI / (1 - SL.HI))).mean() > 0.5  # above the exact sigmoid's bound: fp64 would clamp them
    z = -scene["sdf"][0].astype(np.float64) * 500
    assert (z[cls["saturated_pos"]] >= 100).all() and (z[cls["saturated_neg"]] <= -100).all()
    assert (scene["vis"][cls["vis_below"]] < F32(scene["thr"])).all() and (scene["vis"][cls["vis_at_thr"]] == F32(scene["thr"])).all()
    assert not d["vis"][cls["vis_at_thr"]].any() and d["vis"][cls["vis_above"]].all()
    assert (scene["valid"][cls["invalid"]] == 0).all() and (scene["valid"][~cls["invalid"]] == 1).all()
    assert d["norm_zero"][cls["norm_zero"]].all() and not d["norm_zero"][~cls["norm_zero"]].any()
    g = (scene["sdf"][1::2].astype(np.float64) - scene["sdf"][2::2]) * (0.5 / F32(scene["delta"]))
    nrm = np.linalg.norm(g, axis=0)
    assert (nrm[cls["norm_lt1"]] < 1).all() and (nrm[cls["norm_gt1"]] > 1).all() and (nrm[cls["norm_large"]] > 40).all()


# ---- the float32 transcription of sdf_loss.cuh and its mutations --------------------------------------------------------------------
MUTATIONS = ("no_cap", "cap_grad", "no_tcl", "sp_swap", "sp_thr_on_y", "sp_no_sigmoid", "detach_target", "eik_nl_not_ng",
             "eik_gate_ignored", "no_vis_factor", "vis_ge", "swap_pm", "keep_vy_variants", "bce_mean_over_n", "eik_inv_delta")


def kernel_f32(S, V, gt_on, w_on, vis_on, gated, n_live, mut=(), bce_w=1.0, eik_w=0.1, gs_w=1e-3):
    """sdf_loss_kernel + sdf_point_loss in numpy float32, line by line; rows >= n_live stay NaN (untouched). Returns (loss, v_sdf, v_y1).
    Mutations are one-line mistakes; `>=` at the softplus threshold is not among them: both branches agree there to within an fp32
    ulp (torch's softplus is continuous at its threshold), so no output can tell them apart."""
    f = F32
    n = S["sdf"].shape[1]
    nl = min(n_live, n)
    s = S["sdf"][:V, :nl].astype(f)
    y = S["y1"][0, :nl].astype(f)
    isig, thr, delta, bw, ew, gw = (f(x) for x in (S["isig"], S["thr"], S["delta"], bce_w, eik_w, gs_w))
    lo, hi = f(1e-7), f(1) - f(1e-7)
    vis = S["vis"][:nl].astype(f)
    ok = np.ones(nl, bool)
    if gated:
        ok = (vis > thr) & (S["valid"][:nl] != 0)
    ng = f(max(int(ok.sum()), 1))
    part = np.zeros(nl, f)
    vs0 = np.zeros(nl, f)
    vy = np.zeros(nl, f)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        if gt_on:
            g = S["gt"][:nl].astype(f)
            by = f(100) * y
            lin = (y > f(20)) if "sp_thr_on_y" in mut else (by > f(20))
            spl = np.log1p(np.exp(by)) * f(0.01)
            sp = np.where(lin, spl, y) if "sp_swap" in mut else np.where(lin, y, spl)
            raw = f(1) + sp * isig
            capped = (raw > f(500)) & ("no_cap" not in mut)
            isg = np.where(capped, f(500), raw).astype(f)
            z = -s[0] * isg
            tz = -g * isg
            tsig = f(1) / (f(1) + np.exp(-tz))
            tcl = ((tsig < lo) | (tsig > hi)) & ("no_tcl" not in mut)
            t = np.minimum(np.maximum(tsig, lo), hi)
            bce = np.maximum(z, f(0)) - z * t + np.log1p(np.exp(-np.abs(z)))
            wb = bw / (f(n) if "bce_mean_over_n" in mut else f(nl))
            part += wb * bce
            dz = (f(1) / (f(1) + np.exp(-z)) - t) * wb
            dt = f(0) if "detach_target" in mut else -z * wb
            vs0 += dz * -isg
            d_isg = dz * -s[0] + np.where(tcl, f(0), dt * tsig * (f(1) - tsig) * -g)
            sg = f(1) if "sp_no_sigmoid" in mut else f(1) / (f(1) + np.exp(-by))
            vy = np.where(capped & ("cap_grad" not in mut), f(0), d_isg * isig * np.where(lin, f(1), sg)).astype(f)
        if w_on:
            ww = S["w"][:nl].astype(f) * gw
            if vis_on:
                passed = (vis >= thr) if "vis_ge" in mut else (vis > thr)
                ww = np.where(passed, ww if "no_vis_factor" in mut else ww * vis, f(0))
            if gated:
                ww = np.where(ok, ww, f(0))
            part += f(0.5) * ww * s[0] * s[0]
            vs0 += ww * s[0]
        v_s = [vs0] + [np.zeros(nl, f) for _ in range(V - 1)]
        if V == 7:
            inv2d = (f(1) if "eik_inv_delta" in mut else f(0.5)) / delta
            gx, gy, gz = ((s[1 + 2 * k] - s[2 + 2 * k]) * inv2d for k in range(3))
            nrm = np.sqrt(gx * gx + gy * gy + gz * gz)
            we = ew / (ng if gated and "eik_nl_not_ng" not in mut else f(nl))
            we = np.where(gated & ~ok & ("eik_gate_ignored" not in mut), f(0), we).astype(f)
            part += we * (nrm - f(1)) * (nrm - f(1))
            k = np.where(nrm > 0, f(2) * (nrm - f(1)) / nrm * we * inv2d, f(0)).astype(f)
            sgn = f(-1) if "swap_pm" in mut else f(1)
            for j, gj in enumerate((gx, gy, gz)):
                v_s[1 + 2 * j], v_s[2 + 2 * j] = sgn * k * gj, -sgn * k * gj
    v_sdf = np.full((V, n), np.nan)
    v_y1 = np.full((V, n), np.nan)
    for v in range(V):
        v_sdf[v, :nl] = v_s[v]
        if v == 0 or "keep_vy_variants" not in mut:
            v_y1[v, :nl] = vy if v == 0 else 0.0
    return float(part.astype(np.float64).sum()), v_sdf.reshape(-1), v_y1.reshape(-1)


def _beyond(S, case, n_live, mut=()):
    """(loss beyond?, v_sdf rows beyond, v_y1 rows beyond) of the transcription against the arbiter's bar"""
    V, gt, w, vis, gated = CASES[case]
    R = SC.arbiter(S, V, gt, w, vis, gated, n_live=n_live)
    loss, vs, vy = kernel_f32(S, V, gt, w, vis, gated, n_live, mut)
    nl = R["nl"]
    lb = abs(loss - R["loss"]) > SL.C_ULP * SL.U * SL.loss_scale(R, SL.kernel_sum_steps(S["sdf"].shape[1], nl))
    return lb, int(SL.off_bar(vs, R["v_sdf"], R["v_sdf_scale"]).sum()), int(SL.off_bar(vy, R["v_y1"], R["v_y1_scale"]).sum())


@pytest.mark.parametrize("case", sorted(CASES))
def test_float32_transcription_meets_the_bar(scene, case):
    """the unmutated transcription is within C_ULP 2^-24 scale of the arbiter everywhere: the scales are not too tight for an fp32
    kernel (numpy's float32 exp / log1p stand in for CUDA's expf / log1pf)"""
    n = scene["sdf"].shape[1]
    for n_live in (n, n - DEAD):
        assert _beyond(scene, case, n_live) == (False, 0, 0), case


def test_mutations_move_an_output_beyond_the_bar():
    scenes = [SC.scene(s) for s in SC.ISIGMAS]
    report = []
    for mut in MUTATIONS:
        hits = []
        for S in scenes:
            n = S["sdf"].shape[1]
            for case in sorted(CASES):
                lb, ns, ny = _beyond(S, case, n - DEAD, (mut,))
                if lb or ns or ny:
                    hits.append(f"isig {S['isig']:g} {case}: " + ", ".join(
                        x for x, on in ((f"loss", lb), (f"v_sdf x{ns}", ns), (f"v_y1 x{ny}", ny)) if on))
        report.append(f"{mut}: " + (hits[0] + f" (+{len(hits) - 1} more scene/case pairs)" if hits else "NOT CAUGHT"))
        print(report[-1])
    assert not [r for r in report if r.endswith("NOT CAUGHT")], "\n".join(report)
