"""gssdf_sdf_train in its analytic-eikonal mode (eikonal_mode 1, the reference default) against the fp64 composition of
tests/sdf_train_oracle.py, at the sizes where the persistent kernel's schedule changes shape (tests/sdf_train_shapes.py): several tiles
per CTA, second-order batches gathered from up to seven tiles and flushed inside the tile loop, the weight-gradient accumulators carried
across tiles and batches, live counts on and next to tile boundaries, idle CTAs; and in the arrangements of the training step: world
coordinates with the step's map size and an origin away from zero, the skip-base 7-variant forward into a NaN-filled buffer followed by
the V = 1 train call, device-side live counts, the compacted coupling site and the in-kernel gate, stage [A] and stage [C] accumulating
into the same buffers.

The loss weights, delta, bce_isigma, visible_thr and map size come from a constructed render.GsSdfStep. Inputs keep off the knife
edges of the comparison (sdf_train_oracle.clean_points), so the tolerances are those of DESIGN section 9: loss 1e-4 relative; table
and decoder gradients, total and second-order share, 1e-3 relative L2; dL/dx 5e-4 relative L2 on the rows whose first-order feature
cotangent keeps off an fp16 rounding midpoint (sdf_train_oracle.half_edges; at these batch sizes those cotangents are fp16 subnormals,
where one flipped quantum is a tenth of the value)."""
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import sdf_train_oracle as SO  # noqa: E402
from helpers import assert_close_frac  # noqa: E402
from sdf_train_shapes import CASES, points_per_tile, schedule, summary, targets  # noqa: E402

ORIGIN = (1.5, -2.0, 0.75)
MAP_SIZE = 14.0
HALF_EXTENT = 6.0      # points within origin +- 6 m: x01 in [0.07, 0.93]
TABLE_AMP = 2e-3       # keeps tcnn's fp16 x128 intermediates of the double backward finite (config/base.yaml:12)
BCE_W_RAY, BCE_W_SPLAT = 1.0, 0.0  # the bce_weight arguments of stage [A] and stage [C] in GsSdfStep.step
V_X_SENTINEL = 7.0


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def O(oracle):
    oracle.set_threads(os.cpu_count())
    return oracle


@pytest.fixture(scope="module")
def step(dev):
    """the SDF-loss configuration of the training step, read from the step itself"""
    from gssdf_b200 import render
    cfg = dict(n_levels=16, n_features=2, log2_hashmap_size=19, base_resolution=32, per_level_scale=2.0, hidden_dim=64, n_hidden=3)
    G = render.GsSdfStep(256, 16, 64, 48, dev, 20000, cfg, origin=ORIGIN, map_size=MAP_SIZE)
    assert G.mlp_mode == 1 and G.eik_mode == 1 and G.align_w > 0
    return dict(origin=np.array(G.origin, np.float32), inv_size=G.inv_size, delta=G.delta, bce_isigma=G.bce_isigma, eik_w=G.eik_w,
                gs_w=G.gs_sdf_w, thr=G.vis_thr, align_w=G.align_w)


@pytest.fixture(scope="module")
def sms(dev):
    return torch.cuda.get_device_properties(0).multi_processor_count


class Net:
    """host table / decoder and the device net (mlp_mode 1) in world coordinates; the struct holds raw pointers into the tensors kept here"""

    def __init__(self, O, dev, st, n_hidden, seed):
        from gssdf_b200 import cabi
        rng = np.random.default_rng(seed)
        self.n_hidden = n_hidden
        self.n_params, _ = O.grid_setup()
        self.table = rng.uniform(-TABLE_AMP, TABLE_AMP, self.n_params).astype(np.float32)
        self.mlp = SO.make_mlp(rng, n_hidden)
        self.half = torch.empty(self.n_params, dtype=torch.float16, device=dev)
        cabi.sdf_table_to_half(torch.from_numpy(self.table).to(dev), self.half)
        self.mlp_t = torch.from_numpy(self.mlp).to(dev)
        probe = cabi.sdf_net(self.half, self.mlp_t, n_hidden=n_hidden)
        self.packed = torch.empty(cabi.sdf_mlp_packed_bytes(probe), dtype=torch.uint8, device=dev)
        cabi.sdf_mlp_pack(probe, self.packed)
        self.net = cabi.sdf_net(self.half, self.mlp_t, n_hidden=n_hidden, origin=tuple(st["origin"]), inv_size=st["inv_size"], mlp_mode=1,
                                mlp_packed=self.packed)


def _case(O, net, st, sms, name, site, seed):
    """inputs of one case (live rows off the knife edges, dead rows finite) and the fp64 composition on its live rows"""
    case = CASES[name](sms)
    for what, ok in targets(name, case, sms):
        assert ok, f"{name} on {sms} SMs: {what}"
    n, nl, V = case["n"], case["n_live"], case["V"]
    rng = np.random.default_rng(seed)
    P = SO.clean_points(O, rng, nl, net.table, net.mlp, net.n_hidden, st["origin"], st["inv_size"], st["delta"], HALF_EXTENT)
    x = np.empty((n, 3), np.float32)
    x[:nl] = P["xw"]
    x[nl:] = st["origin"] + rng.uniform(-HALF_EXTENT, HALF_EXTENT, (n - nl, 3))
    c = dict(name=name, site=site, n=n, n_live=nl, V=V, x=x)
    kw = dict(inv_size=st["inv_size"], delta=st["delta"], eikonal_weight=st["eik_w"], align_weight=st["align_w"], n_live=nl,
              bce_isigma=st["bce_isigma"])
    if site == "ray":
        c["gt"] = rng.uniform(-0.3, 0.3, n).astype(np.float32)
        R = SO.compose(O, P, net.table, net.mlp, net.n_hidden, gt=c["gt"][:nl], bce_weight=BCE_W_RAY, **kw)
    elif site == "compact":  # rows of the compacted gate: weights already multiplied by the visibility, every live row passed the gate
        c["w"] = rng.uniform(0.1, 1.0, n).astype(np.float32)
        R = SO.compose(O, P, net.table, net.mlp, net.n_hidden, weights=c["w"][:nl], gs_sdf_weight=st["gs_w"], bce_weight=BCE_W_SPLAT, **kw)
    else:  # "gated": the in-kernel gate over all live rows
        c["w"] = rng.uniform(0.1, 1.0, n).astype(np.float32)
        c["vis"] = rng.uniform(0.0, 3 * st["thr"], n).astype(np.float32)
        c["valid"] = (rng.uniform(0, 1, n) > 0.2).astype(np.uint8)
        R = SO.compose(O, P, net.table, net.mlp, net.n_hidden, weights=c["w"][:nl], gs_sdf_weight=st["gs_w"], bce_weight=BCE_W_SPLAT,
                       visibilities=c["vis"][:nl], valid_mask=c["valid"][:nl], visible_thr=st["thr"], gated=True, **kw)
        assert 0.3 * nl < R["n_gate"] < 0.8 * nl
    c["sched"] = summary(schedule(n, V, sms, nl))
    return c, R


def _run(net, st, c, dev, bufs=None, device_n_live=True):
    """the case's calls in the step's arrangement; `bufs` = (loss, table_grad, mlp_grad) to accumulate into"""
    from gssdf_b200 import cabi
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    n, V = c["n"], c["V"]
    loss, tg, mg = bufs if bufs is not None else (torch.zeros(1, device=dev), torch.zeros(net.n_params, device=dev),
                                                   torch.zeros(len(net.mlp), device=dev))
    x = t(c["x"])
    nl = torch.tensor([c["n_live"]], dtype=torch.int32, device=dev) if device_n_live else None
    vx = torch.full((n, 3), V_X_SENTINEL, device=dev) if c["site"] != "ray" or V == 7 else None
    sdf7 = None
    if V == 1:  # 7-variant forward without the base variant into a NaN-filled buffer: the train call must read only variants 1..6
        sdf7 = torch.full((7 * n,), float("nan"), device=dev)
        cabi.sdf_fwd(net.net, x, sdf7, None, None, n_variants=7, delta=st["delta"], skip_base_variant=True, n_live=nl)
    kw = dict(n_live=nl, eikonal_mode=1, align_weight=st["align_w"], sdf_variants=sdf7)
    if c["site"] == "ray":
        cabi.sdf_train(net.net, x, V, st["delta"], t(c["gt"]), None, st["bce_isigma"], BCE_W_RAY, st["eik_w"], 0.0, loss, tg, mg, vx, **kw)
    elif c["site"] == "compact":
        cabi.sdf_train(net.net, x, V, st["delta"], None, t(c["w"]), st["bce_isigma"], BCE_W_SPLAT, st["eik_w"], st["gs_w"], loss, tg, mg, vx,
                       **kw)
    else:
        vis, valid = t(c["vis"]), t(c["valid"])
        ng = torch.zeros(1, dtype=torch.int32, device=dev)
        cabi.sdf_gate_count(n, ng, visibilities=vis, visible_thr=st["thr"], valid_mask=valid, n_live=nl)
        cabi.sdf_train(net.net, x, V, st["delta"], None, t(c["w"]), st["bce_isigma"], BCE_W_SPLAT, st["eik_w"], st["gs_w"], loss, tg, mg, vx,
                       visibilities=vis, visible_thr=st["thr"], valid_mask=valid, n_gate=ng, **kw)
        c["n_gate_dev"] = ng
    torch.cuda.synchronize()
    return loss, tg, mg, vx


def _check(c, R, loss, tg, mg, vx, prefill=None):
    """loss 1e-4; table / decoder gradients 1e-3 relative L2, in total and their second-order share; decoder gradient elementwise;
    dL/dx 5e-4 relative L2 on the live rows off an fp16 edge and untouched beyond n_live"""
    lg, tgc, mgc = float(loss[0]), tg.cpu().numpy().astype(np.float64), mg.cpu().numpy().astype(np.float64)
    if prefill is not None:
        lg, tgc, mgc = lg - prefill[0], tgc - prefill[1], mgc - prefill[2]
    assert np.isfinite(lg) and np.isfinite(tgc).all() and np.isfinite(mgc).all()
    r_tg = R["table1"] + R["table2"]
    e_l = abs(lg - R["loss"]) / abs(R["loss"])
    e_m, e_t = rel(mgc, R["mlp"]), rel(tgc, r_tg)
    e_m2, e_t2 = rel(mgc - R["mlp1"], R["mlp2"]), rel(tgc - R["table1"], R["table2"])
    bad = np.abs(mgc - R["mlp"]) > 1e-3 * np.abs(R["mlp"]) + 1e-4 * np.abs(R["mlp"]).max()
    msg = (f"SDFTRAIN {c['name']}/{c['site']} V={c['V']} n={c['n']} live={c['n_live']}: loss {e_l:.1e}; mlp {e_m:.1e} (2nd {e_m2:.1e}, "
           f"elementwise off {bad.mean():.1e}); table {e_t:.1e} (2nd {e_t2:.1e})")
    if vx is not None:
        v = vx.cpu().numpy()
        e_v_all = rel(v[:c["n_live"]], R["v_x"])
        off = ~R["v_x_edge"]
        e_v = rel(v[:c["n_live"]][off], R["v_x"][off])
        msg += f"; v_x {e_v:.1e} (all rows {e_v_all:.1e}, {R['v_x_edge'].mean():.1%} on an fp16 edge, |v_x| {np.linalg.norm(R['v_x']):.1e})"
    print(msg + f"; 2nd/1st mlp norm {np.linalg.norm(R['mlp2']) / max(np.linalg.norm(R['mlp1']), 1e-300):.1e}")
    assert np.linalg.norm(R["mlp2"]) > 1e-3 * np.linalg.norm(R["mlp1"])  # the second-order part is a visible share
    assert e_l <= 1e-4, msg
    assert e_m <= 1e-3 and e_t <= 1e-3, msg
    assert e_m2 <= 1e-3 and e_t2 <= 1e-3, msg
    assert_close_frac(mgc, R["mlp"], 1e-3, 1e-4 * np.abs(R["mlp"]).max(), 1e-3, "mlp grad")
    if vx is not None:
        assert np.isfinite(v).all()
        assert R["v_x_edge"].mean() < 0.3, msg
        assert e_v <= 5e-4, msg
        assert (v[c["n_live"]:] == V_X_SENTINEL).all(), "dL/dx written beyond n_live"


# ------------------------------------------------------------------------------------------------------------------------------
# (a) V = 7 ray samples, ~20 k points: a full 7-tile batch flushed inside the tile loop, then a partial one; every decoder depth
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_hidden", [0, 1, 2, 3])
def test_full_batches_v7_every_depth(O, dev, step, sms, n_hidden):
    net = Net(O, dev, step, n_hidden, seed=100 + n_hidden)
    c, R = _case(O, net, step, sms, "full_batches_v7", "ray", seed=n_hidden)
    full = points_per_tile(7) * 7
    assert all(k[0] == full and len(k) == 2 for k in c["sched"]), c["sched"]
    _check(c, R, *_run(net, step, c, dev))


# ------------------------------------------------------------------------------------------------------------------------------
# (b) + (c): the two train calls of the step, one decoder, the same gradient buffers
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def step_net(O, dev, step):
    return Net(O, dev, step, 3, seed=7)


@pytest.fixture(scope="module")
def ray_case(O, step_net, step, sms):
    return _case(O, step_net, step, sms, "ray_stage", "ray", seed=11)


@pytest.fixture(scope="module")
def coupling_case(O, step_net, step, sms):
    return _case(O, step_net, step, sms, "coupling_compact", "compact", seed=12)


def test_ray_stage_arrangement(dev, step, step_net, ray_case):
    """(b) stage [A]: 49 152-row buffer, ~30 k live rows (device count), skip-base 7-variant forward then V = 1 with sdf_variants"""
    c, R = ray_case
    _check(c, R, *_run(step_net, step, c, dev))


def test_coupling_stage_compact_arrangement(dev, step, step_net, coupling_case):
    """(c) stage [C] on the compacted gated samples: ~120 k rows, n_live = n_gate ~53 k, weights x vis, gs_sdf, no BCE, dL/dx"""
    c, R = coupling_case
    _check(c, R, *_run(step_net, step, c, dev))


def test_ray_then_coupling_accumulate(dev, step, step_net, ray_case, coupling_case):
    """(b) then (c) into the same, pre-filled loss and gradient buffers == the pre-filled values + the sum of both compositions"""
    (cb, Rb), (cc, Rc) = ray_case, coupling_case
    rng = np.random.default_rng(3)
    R = SO.add(Rb, Rc)
    p_loss = np.float32(0.375)
    p_tg = (rng.standard_normal(step_net.n_params) * np.abs(Rb["table1"]).max() * 0.1).astype(np.float32)
    p_mg = (rng.standard_normal(len(step_net.mlp)) * np.abs(R["mlp"]).max()).astype(np.float32)
    bufs = (torch.tensor([p_loss], device=dev), torch.from_numpy(p_tg).to(dev), torch.from_numpy(p_mg).to(dev))
    _run(step_net, step, cb, dev, bufs)
    loss, tg, mg, vx = _run(step_net, step, cc, dev, bufs)
    _check(dict(cc, name="ray_then_coupling"), dict(R, v_x=Rc["v_x"], v_x_edge=Rc["v_x_edge"]), loss, tg, mg, vx,
           prefill=(float(p_loss), p_tg.astype(np.float64), p_mg.astype(np.float64)))


# ------------------------------------------------------------------------------------------------------------------------------
# (d) in-kernel gate, (e) live-count edges, (f) six tiles per CTA
# ------------------------------------------------------------------------------------------------------------------------------
def test_gate_in_kernel_multi_tile_batches(O, dev, step, step_net, sms):
    """(d) visibilities + valid mask + n_gate on the full batch, V = 7, four or five tiles in every batch"""
    c, R = _case(O, step_net, step, sms, "gate_in_kernel", "gated", seed=13)
    out = _run(step_net, step, c, dev)
    assert int(c["n_gate_dev"][0]) == R["n_gate"]
    _check(c, R, *out)


@pytest.mark.parametrize("name,V", [("live_boundary", 7), ("live_boundary_plus_one", 7), ("idle_ctas", 1)])
def test_live_count_edges(O, dev, step, step_net, sms, name, V):
    """(e) n_live on a tile boundary and one past it (V = 7), and a large buffer with fewer live tiles than SMs (V = 1)"""
    c, R = _case(O, step_net, step, sms, name, "ray", seed=20 + len(name))
    assert c["V"] == V
    _check(c, R, *_run(step_net, step, c, dev))


def test_six_tiles_per_cta(O, dev, step, step_net, sms):
    """(f) ~100 k points, V = 1 with the 7-variant forward, no live count: every tile its own batch, five or six per CTA"""
    c, R = _case(O, step_net, step, sms, "six_tiles", "ray", seed=30)
    _check(c, R, *_run(step_net, step, c, dev, device_n_live=False))
