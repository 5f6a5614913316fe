"""Host-side checks (no GPU) for the analytic-eikonal SDF train tests: the schedule mirror of tests/sdf_train_shapes.py against schedules
worked out by hand, every GPU case reaching its schedule target on both H100 variants, and the glue of the fp64 composition in
tests/sdf_train_oracle.py (world -> x01 coordinates, the gate and its means, the eikonal / align cotangent with respect to the x01
gradient) against torch.autograd in fp64. The oracle chains the composition is built from are pinned in test_sdf_oracle.py."""
import numpy as np
import pytest

import sdf_train_oracle as SO
from sdf_train_shapes import CASES, H100_SMS, schedule, summary, targets

torch = pytest.importorskip("torch")


def test_schedule_mirror_reproduces_hand_counts():
    # 1500 points x 7 variants: 84 tiles of 18 points, one CTA each; the last tile holds 1500 - 83 * 18 = 6 points
    c = schedule(1500, 7, 132)
    assert len(c) == 84 and all(len(x["tiles"]) == 1 for x in c)
    assert summary(c) == {(18,): 83, (6,): 1}
    # 20 000 x 7 on 132 SMs: 1112 tiles; CTAs 0..55 run 9 tiles, the others 8; tile 1111 (CTA 55) holds 2 points
    c = schedule(20000, 7, 132)
    assert sum(len(x["tiles"]) for x in c) == 1112 and len(c) == 132
    assert summary(c) == {(126, 18): 76, (126, 36): 55, (126, 20): 1}
    # 30 000 live of 49 152 x 1: 235 live tiles (the last with 48 points) on 132 CTAs; a batch is one tile, so every tile flushes
    c = schedule(49152, 1, 132, n_live=30000)
    assert sum(1 for x in c if len(x["tiles"]) == 2) == 103
    assert summary(c) == {(128, 128): 102, (128, 48): 1, (128,): 29}
    # no live point: every CTA idle
    assert summary(schedule(49152, 1, 132, n_live=0)) == {(): 132}


def test_schedule_mirror_conserves_points():
    rng = np.random.default_rng(0)
    for _ in range(200):
        V = int(rng.choice([1, 7]))
        n = int(rng.integers(1, 40000))
        nl = int(rng.integers(0, n + 1))
        sms = int(rng.choice([132, 114, 7]))
        c = schedule(n, V, sms, nl)
        assert sum(sum(x["flushes"]) for x in c) == nl
        assert all(0 < f <= 128 for x in c for f in x["flushes"])


@pytest.mark.parametrize("sms", H100_SMS)
@pytest.mark.parametrize("name", sorted(CASES))
def test_gpu_cases_reach_their_schedule(name, sms):
    case = CASES[name](sms)
    assert 0 < case["n_live"] <= case["n"]
    for what, ok in targets(name, case, sms):
        assert ok, f"{name} on {sms} SMs: {what} ({case})"


# ------------------------------------------------------------------------------------------------------------------------------
def test_world_to_x01_is_the_kernels_float32_arithmetic():
    rng = np.random.default_rng(1)
    origin, inv = np.array([1.5, -2.0, 0.75], np.float32), 1.0 / 14.0
    xw = (origin + rng.uniform(-6, 6, (5000, 3))).astype(np.float32)
    # two float32 roundings, as separate operations: (x - origin) * inv, then + 0.5
    t = (torch.from_numpy(xw) - torch.from_numpy(origin)) * torch.tensor(inv, dtype=torch.float32) + 0.5
    assert np.array_equal(SO.world_to_x01(xw, origin, inv), t.numpy())
    # variants: +-delta on one world coordinate first, in float32
    v = SO.variant_world(xw, 0.1)
    assert v.dtype == np.float32 and v.shape == (6, 5000, 3)
    for k in range(6):
        d = k // 2
        want = xw.copy()
        want[:, d] = (want[:, d] + (np.float32(-0.1) if k % 2 else np.float32(0.1))).astype(np.float32)
        assert np.array_equal(v[k], want)
    assert np.array_equal(SO.world_to_x01(xw, origin, 0.0), xw)


def _torch_second_order(g01, gnum, isz, eik_w, align_w, ok, nl):
    g = g01 * isz
    nrm = g.norm(dim=1)
    okf = ok.double()
    loss = eik_w * (okf * (nrm - 1) ** 2).sum() / nl
    if gnum is not None:
        loss = loss + align_w * (okf[:, None] * (g - gnum).abs()).sum() / (3 * nl)
    return loss


@pytest.mark.parametrize("gated,align", [(False, True), (True, True), (True, False)])
def test_second_order_cotangent_matches_autograd(gated, align):
    rng = np.random.default_rng(2 + gated + 2 * align)
    n, isz, eik_w, align_w, thr = 300, 1.0 / 14.0, 0.1, 0.1, 0.1
    g01 = rng.standard_normal((n, 3)) * 14.0
    gnum = rng.standard_normal((n, 3)) if align else None
    vis = rng.uniform(0, 0.3, n).astype(np.float32)
    valid = (rng.uniform(0, 1, n) > 0.2).astype(np.uint8)
    n_live = 250  # rows beyond n_live are not part of the composition
    ok, nl = SO.gate(n_live, vis, valid, thr, gated)
    assert nl == (int(((vis[:n_live] > thr) & (valid[:n_live] != 0)).sum()) if gated else n_live)
    loss, c01 = SO.second_order_terms(g01[:n_live], None if gnum is None else gnum[:n_live], isz, eik_w, align_w, ok, nl)
    G = torch.tensor(g01[:n_live], dtype=torch.float64, requires_grad=True)
    T = _torch_second_order(G, None if gnum is None else torch.tensor(gnum[:n_live]), isz, eik_w, align_w, torch.from_numpy(ok), nl)
    T.backward()
    assert abs(loss - T.item()) <= 1e-12 * abs(T.item())
    assert np.allclose(c01, G.grad.numpy(), rtol=1e-12, atol=1e-18)
    assert (c01[~ok] == 0).all() and np.abs(c01[ok]).min() > 0


def test_coupling_weights_and_gate_match_autograd(oracle):
    """first-order coupling term 0.5 gs_sdf_weight w vis s^2 (vis > thr, gate passed) through oracle.sdf_losses, dL/ds vs autograd"""
    O = oracle
    rng = np.random.default_rng(5)
    n, gs_w, thr = 400, 1e-3, 0.1
    s = rng.standard_normal(n)
    w = rng.uniform(0.2, 1.0, n).astype(np.float32)
    vis = rng.uniform(0, 0.3, n).astype(np.float32)
    valid = (rng.uniform(0, 1, n) > 0.3).astype(np.uint8)
    for gated in (False, True):
        ok, _ = SO.gate(n, vis, valid, thr, gated)
        we = SO.coupling_weights(w, gs_w, vis, thr, ok)
        loss, v_s, v_y = O.sdf_losses(s, np.zeros(n), n, 1, weights=we, gs_sdf_weight=1.0, eikonal_weight=0.0)
        S = torch.tensor(s, requires_grad=True)
        keep = torch.from_numpy(vis > thr) & (torch.from_numpy(valid != 0) if gated else torch.ones(n, dtype=torch.bool))
        T = (0.5 * gs_w * torch.from_numpy(w).double() * torch.from_numpy(vis).double() * S ** 2 * keep.double()).sum()
        T.backward()
        assert abs(loss - T.item()) <= 1e-12 * abs(T.item())
        assert np.allclose(v_s, S.grad.numpy(), rtol=1e-12, atol=0) and not v_y.any()


def test_composition_on_the_host(oracle):
    """the whole composition on a few clean points: finite, shares add up, the eikonal part vanishes without weight, the world-unit
    dL/dx is the x01 one times inv_size, and the builder keeps only points off the knife edges"""
    rng = np.random.default_rng(6)
    n_params, _ = oracle.grid_setup()
    table = rng.uniform(-2e-3, 2e-3, n_params).astype(np.float32)
    mlp = SO.make_mlp(rng, 1)
    origin, isz, delta = np.array([1.5, -2.0, 0.75], np.float32), 1.0 / 14.0, 0.1
    P = SO.clean_points(oracle, rng, 200, table, mlp, 1, origin, isz, delta, 6.0)
    assert len(P["sdf"]) == 200 and not SO.knife_edges(P, isz).any()
    gt = rng.uniform(-0.1, 0.1, 200).astype(np.float32)
    R = SO.compose(oracle, P, table, mlp, 1, isz, delta, 0.1, 0.1, 200, gt=gt, bce_isigma=10.0, bce_weight=1.0)
    assert np.allclose(R["mlp"], R["mlp1"] + R["mlp2"]) and abs(R["loss"] - R["loss1"] - R["loss2"]) <= 1e-15
    assert np.linalg.norm(R["mlp2"]) > 1e-3 * np.linalg.norm(R["mlp1"])
    l1, v_s, v_y = oracle.sdf_losses(P["sdf"], P["y1"], 200, 1, gt_sdf=gt, bce_isigma=10.0, bce_weight=1.0, eikonal_weight=0.0)
    _, _, dx = oracle.sdf_bwd(P["x01"], table, mlp, v_s, v_y, 64, 1)
    assert np.array_equal(R["v_x"], np.asarray(dx, np.float64) * isz) and R["loss1"] == l1
    R0 = SO.compose(oracle, P, table, mlp, 1, isz, delta, 0.0, 0.0, 200, gt=gt, bce_isigma=10.0, bce_weight=1.0)
    assert R0["loss2"] == 0 and not R0["mlp2"].any() and not R0["table2"].any()
