"""GPU parity of the SDF branch (fused hash-grid + decoder MLP, first order) vs the CPU oracle.
Features are compared EXACTLY (they are fp16 values produced with the same rounding points); the fp32 MLP
outputs and all gradients at 1e-4 relative to the fp64 oracle chain (with an fp32 absolute floor)."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import sdf_train_oracle as SO  # noqa: E402
from helpers import assert_close_frac  # noqa: E402


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _mlp(rng, hidden, n_hidden, in_dim=32):
    dims = [in_dim] + [hidden] * (1 + n_hidden) + [2]
    ps = []
    for k, o in zip(dims[:-1], dims[1:]):
        b = 1 / np.sqrt(k)
        ps += [rng.uniform(-b, b, o * k), rng.uniform(-b, b, o)]
    return np.concatenate(ps).astype(np.float32)


def _relu_ties(feat, mlp, hidden, n_hidden, eps=2e-6):
    """Rows with a hidden pre-activation within `eps` of zero (fp64): relu' is discontinuous there, so an fp32-grade
    implementation may legitimately pick the other side than the fp64 oracle. Their cotangents are zeroed in the tests."""
    a, o, K = feat.astype(np.float64), 0, feat.shape[1]
    tie = np.zeros(len(feat), bool)
    for _ in range(1 + n_hidden):
        W = mlp[o:o + hidden * K].reshape(hidden, K).astype(np.float64)
        b = mlp[o + hidden * K:o + hidden * K + hidden].astype(np.float64)
        o += hidden * K + hidden
        z = a @ W.T + b
        tie |= (np.abs(z) < eps).any(1)
        a, K = np.maximum(z, 0), hidden
    return tie


@pytest.mark.parametrize("n,hidden,n_hidden", [(5000, 64, 3), (777, 32, 1), (130, 64, 0)])
def test_sdf_fwd_bwd(oracle, n, hidden, n_hidden):
    from gssdf_b200 import cabi
    dev = _dev()
    rng = np.random.default_rng(n)
    n_params, _ = oracle.grid_setup()
    table = rng.uniform(-0.5, 0.5, n_params).astype(np.float32)  # SURVEY 8d: U(-0.5,0.5) for parity
    mlp = _mlp(rng, hidden, n_hidden)
    x = rng.uniform(0.02, 0.98, (n, 3)).astype(np.float32)
    x[:64] = rng.choice(np.array([0.0, 1.0, 0.99, 0.985, 1.02, -0.01], np.float32), (64, 3))  # cube faces / slightly outside: index wrap
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    tab, half = t(table), torch.empty(n_params, dtype=torch.float16, device=dev)
    cabi.sdf_table_to_half(tab, half)
    assert np.array_equal(half.cpu().numpy().view(np.uint16), oracle.f32_to_f16_bits(table))
    mlp_t = t(mlp)  # keep alive: the net struct only holds raw pointers
    net = cabi.sdf_net(half, mlp_t, hidden_dim=hidden, n_hidden=n_hidden)
    assert cabi.sdf_table_params(net) == n_params and cabi.sdf_mlp_params(net) == len(mlp)
    sdf, y1, feat = torch.empty(n, device=dev), torch.empty(n, device=dev), torch.empty(n, 32, device=dev)
    cabi.sdf_fwd(net, t(x), sdf, y1, feat)
    r_sdf, r_y1, r_feat = oracle.sdf_fwd(x, table, mlp, hidden, n_hidden)
    assert np.array_equal(feat.cpu().numpy(), r_feat), "hash-grid features must be bit-identical (fp16 rounding points)"
    assert_close_frac(sdf.cpu().numpy(), r_sdf, 1e-4, 1e-5, 0.0, "sdf")
    assert_close_frac(y1.cpu().numpy(), r_y1, 1e-4, 1e-5, 0.0, "y1")
    # backward
    v_sdf, v_y1 = rng.standard_normal(n).astype(np.float32), rng.standard_normal(n).astype(np.float32)
    tie = _relu_ties(r_feat, mlp, hidden, n_hidden)
    v_sdf[tie], v_y1[tie] = 0, 0
    tg, mg, vx = torch.zeros(n_params, device=dev), torch.zeros(len(mlp), device=dev), torch.empty(n, 3, device=dev)
    cabi.sdf_bwd(net, t(x), t(v_sdf), t(v_y1), tg, mg, vx)
    r_tg, r_mg, r_vx = oracle.sdf_bwd(x, table, mlp, v_sdf, v_y1, hidden, n_hidden)
    assert_close_frac(mg.cpu().numpy(), r_mg, 1e-4, 1e-5 * np.abs(r_mg).max(), 0.0, "mlp grad")
    # the cotangent reaching the encoding is rounded to fp16 (x128) in both; an fp32-vs-fp64 difference of the MLP
    # backward can flip that rounding by one fp16 ulp (2^-11 relative) on isolated entries
    assert_close_frac(tg.cpu().numpy(), r_tg, 2e-3, 1e-5 * np.abs(r_tg).max(), 1e-3, "table grad")
    assert np.linalg.norm(tg.cpu().numpy() - r_tg) <= 2e-4 * np.linalg.norm(r_tg)
    assert_close_frac(vx.cpu().numpy(), r_vx, 2e-3, 1e-4 * np.abs(r_vx).max(), 1e-3, "v_x")
    assert np.linalg.norm(vx.cpu().numpy() - r_vx) <= 5e-4 * np.linalg.norm(r_vx)


def test_sdf_mirror_api_autograd_and_numerical_gradient(oracle):
    from gssdf_b200 import sdf as sdfmod
    dev = _dev()
    net = sdfmod.SdfNet(dev, map_size=14.0, origin=(0.5, -0.25, 0.1))
    with torch.no_grad():
        net.params_.uniform_(-0.5, 0.5)
    xyz = (torch.rand(3000, 3, device=dev) - 0.5) * 10 + torch.tensor([0.5, -0.25, 0.1], device=dev)
    xyz.requires_grad_(True)
    sdf, isigma = net.get_sdf(xyz)
    assert sdf.shape == (3000, 1) and isigma.shape == (3000, 1) and (isigma >= 1).all()
    (sdf.square().sum() + isigma.sum()).backward()
    assert net.params_.grad is not None and net.decoder_.grad is not None and xyz.grad is not None
    assert torch.isfinite(net.params_.grad).all() and net.params_.grad.abs().sum() > 0
    # same arithmetic as the kernel and the reference (SubMap::xyz_to_zp1_pts as separate fp32 ops: fl(fl((x - pos) * inv) + 0.5));
    # the fp16 grid amplifies 1-ulp input changes
    d32 = (xyz.detach().cpu().numpy() - np.array([0.5, -0.25, 0.1], np.float32)).astype(np.float32)
    x01 = ((d32 * np.float32(1.0 / 14.0)).astype(np.float32) + np.float32(0.5)).astype(np.float32)
    r_sdf, _, _ = oracle.sdf_fwd(x01, net.params_.detach().cpu().numpy(), net.decoder_.detach().cpu().numpy())
    assert_close_frac(sdf.detach().cpu().numpy()[:, 0], r_sdf, 2e-4, 2e-5, 2e-3, "sdf (world coords)")  # x01 rounding differs by an ulp
    g = net.get_gradient_numerical(xyz.detach(), 0.05)
    assert g.shape == (3000, 3) and torch.isfinite(g).all()


def test_sdf_error_conventions():
    from gssdf_b200 import cabi
    dev = _dev()
    z = torch.zeros(16, device=dev)
    with pytest.raises(Exception, match="n_levels 16"):
        cabi.sdf_fwd(cabi.sdf_net(z.half(), z, n_levels=8), torch.zeros(4, 3, device=dev), torch.zeros(4, device=dev))
    cabi.sdf_fwd(cabi.sdf_net(z.half(), z), torch.zeros(0, 3, device=dev), torch.zeros(0, device=dev))  # n == 0: legal no-op


def test_sdf_variants_and_losses(oracle):
    """7-variant evaluation (base + 6 numerical-gradient offsets) and the fused loss kernel vs numpy fp64."""
    from gssdf_b200 import cabi
    dev = _dev()
    rng = np.random.default_rng(11)
    n, delta = 2000, 0.01
    n_params, _ = oracle.grid_setup()
    table = rng.uniform(-0.5, 0.5, n_params).astype(np.float32)
    mlp = _mlp(rng, 64, 3)
    x = rng.uniform(0.05, 0.95, (n, 3)).astype(np.float32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    tab, half, mlp_t, xt = t(table), torch.empty(n_params, dtype=torch.float16, device=dev), t(mlp), t(x)
    cabi.sdf_table_to_half(tab, half)
    net = cabi.sdf_net(half, mlp_t)
    sdf, y1 = torch.empty(7 * n, device=dev), torch.empty(7 * n, device=dev)
    cabi.sdf_fwd(net, xt, sdf, y1, None, n_variants=7, delta=delta)
    offs = np.array([[0, 0, 0], [1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.float32) * np.float32(delta)
    pts = (x[None] + offs[:, None]).reshape(-1, 3).astype(np.float32)
    r_sdf, r_y1, _ = oracle.sdf_fwd(pts, table, mlp)
    assert_close_frac(sdf.cpu().numpy(), r_sdf, 1e-4, 1e-5, 0.0, "sdf x7")
    # losses (ray-sample flavour: bce + eikonal ; splat-sample flavour: gs_sdf + eikonal)
    gt = (rng.standard_normal(n) * 0.05).astype(np.float32)
    w = rng.uniform(0, 1, n).astype(np.float32)
    for kw in (dict(gt_sdf=gt, weights=None), dict(gt_sdf=None, weights=w)):
        loss = torch.zeros(1, device=dev)
        v_s, v_y = torch.empty(7 * n, device=dev), torch.empty(7 * n, device=dev)
        cabi.sdf_loss(n, 7, sdf, y1, t(kw["gt_sdf"]) if kw["gt_sdf"] is not None else None,
                      t(kw["weights"]) if kw["weights"] is not None else None, 10.0, 1.0, 0.1, 1e-3, delta, loss, v_s, v_y)
        r_loss, r_vs, r_vy = oracle.sdf_losses(sdf.cpu().numpy(), y1.cpu().numpy(), n, 7, kw["gt_sdf"], kw["weights"], 10.0, 1.0, 0.1,
                                               1e-3, delta)
        assert abs(float(loss) - r_loss) <= 1e-4 * abs(r_loss) + 1e-7
        assert_close_frac(v_s.cpu().numpy(), r_vs, 1e-3, 1e-5 * np.abs(r_vs).max(), 0.0, "v_sdf")
        assert_close_frac(v_y.cpu().numpy(), r_vy, 1e-3, 1e-5 * max(np.abs(r_vy).max(), 1e-12), 0.0, "v_y1")
    # backward through all 7 variants: gradient to x only through variant 0
    tg, mg, vx = torch.zeros(n_params, device=dev), torch.zeros(len(mlp), device=dev), torch.empty(n, 3, device=dev)
    cabi.sdf_bwd(net, xt, v_s, v_y, tg, mg, vx, n_variants=7, delta=delta)
    r_tg, r_mg, r_vx = oracle.sdf_bwd(pts, table, mlp, v_s.cpu().numpy(), v_y.cpu().numpy())
    assert_close_frac(mg.cpu().numpy(), r_mg, 1e-4, 5e-5 * np.abs(r_mg).max(), 1e-3, "mlp grad x7")  # fp32 sums over 14 k points
    assert np.linalg.norm(mg.cpu().numpy() - r_mg) <= 1e-4 * np.linalg.norm(r_mg)
    # the mean-normalised cotangents here are ~1e-6: the binding casts dL/dy to fp16 BEFORE the x128 loss scale
    # (TB/tcnn_binding.cpp:133), i.e. into the fp16 subnormal range (quantum 6e-8), where an fp32-vs-fp64 ulp of the MLP
    # backward flips whole quanta -> the comparison is only meaningful at the ~1e-3 level
    assert np.linalg.norm(tg.cpu().numpy() - r_tg) <= 2e-3 * np.linalg.norm(r_tg)
    assert np.linalg.norm(vx.cpu().numpy() - r_vx[:n]) <= 2e-3 * np.linalg.norm(r_vx[:n])


_KEEP = []


def _tc_net(cabi, half, mlp_t, n_hidden):
    """mlp_mode=1 net: pre-split weight image (gssdf_sdf_mlp_pack); the struct holds raw pointers -> keep the tensors alive."""
    probe = cabi.sdf_net(half, mlp_t, hidden_dim=64, n_hidden=n_hidden)
    packed = torch.empty(cabi.sdf_mlp_packed_bytes(probe), dtype=torch.uint8, device=mlp_t.device)
    cabi.sdf_mlp_pack(probe, packed)
    _KEEP.append(packed)
    return cabi.sdf_net(half, mlp_t, hidden_dim=64, n_hidden=n_hidden, mlp_mode=1, mlp_packed=packed)


@pytest.mark.parametrize("n,n_hidden,variants", [(5000, 3, 1), (1000, 1, 7), (130, 0, 1)])
def test_sdf_fwd_tensor_core_path(oracle, n, n_hidden, variants):
    """mlp_mode=1: decoder on the Hopper tensor cores (wgmma, bf16 hi/mid split, fp32 accumulate in registers).
    Features stay bit-exact; sdf/y1 within 1e-4 relative (+1e-5 absolute, the same bar as the fp32 CUDA-core path) of the fp64
    oracle: the forward uses a 3-term bf16 split of both operands (24 significant bits)."""
    from gssdf_b200 import cabi
    dev = _dev()
    rng = np.random.default_rng(n + 1)
    n_params, _ = oracle.grid_setup()
    table = rng.uniform(-0.5, 0.5, n_params).astype(np.float32)
    mlp = _mlp(rng, 64, n_hidden)
    x = rng.uniform(0.02, 0.98, (n, 3)).astype(np.float32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    tab, half, mlp_t, xt = t(table), torch.empty(n_params, dtype=torch.float16, device=dev), t(mlp), t(x)
    cabi.sdf_table_to_half(tab, half)
    net = _tc_net(cabi, half, mlp_t, n_hidden)
    delta = 0.01
    sdf, y1, feat = torch.empty(variants * n, device=dev), torch.empty(variants * n, device=dev), torch.empty(variants * n, 32, device=dev)
    cabi.sdf_fwd(net, xt, sdf, y1, feat, n_variants=variants, delta=delta)
    torch.cuda.synchronize()
    offs = np.array([[0, 0, 0], [1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.float32)[:variants] * np.float32(delta)
    pts = (x[None] + offs[:, None]).reshape(-1, 3).astype(np.float32)
    r_sdf, r_y1, r_feat = oracle.sdf_fwd(pts, table, mlp, 64, n_hidden)
    assert np.array_equal(feat.cpu().numpy(), r_feat)
    assert_close_frac(sdf.cpu().numpy(), r_sdf, 1e-4, 1e-5, 0.0, "sdf (tensor cores)")
    assert_close_frac(y1.cpu().numpy(), r_y1, 1e-4, 1e-5, 0.0, "y1 (tensor cores)")


@pytest.mark.parametrize("n,n_hidden,variants", [(5000, 3, 1), (40000, 3, 1), (1000, 1, 7), (130, 0, 1)])
def test_sdf_bwd_tensor_core_path(oracle, n, n_hidden, variants):
    """mlp_mode=1 backward: forward recompute, dL/da GEMMs and the weight-gradient GEMMs (accumulated in registers across the
    persistent CTA's tiles) all on wgmma; compared with the fp64 oracle chain at the same tolerances as the SIMT path
    (a slightly larger absolute floor for the 16-bit operand split)."""
    from gssdf_b200 import cabi
    dev = _dev()
    rng = np.random.default_rng(7 * n + 3)
    n_params, _ = oracle.grid_setup()
    table = rng.uniform(-0.5, 0.5, n_params).astype(np.float32)
    mlp = _mlp(rng, 64, n_hidden)
    x = rng.uniform(0.02, 0.98, (n, 3)).astype(np.float32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    tab, half, mlp_t, xt = t(table), torch.empty(n_params, dtype=torch.float16, device=dev), t(mlp), t(x)
    cabi.sdf_table_to_half(tab, half)
    net = _tc_net(cabi, half, mlp_t, n_hidden)
    delta = 0.01
    offs = np.array([[0, 0, 0], [1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.float32)[:variants] * np.float32(delta)
    pts = (x[None] + offs[:, None]).reshape(-1, 3).astype(np.float32)
    v_sdf, v_y1 = rng.standard_normal(variants * n).astype(np.float32), rng.standard_normal(variants * n).astype(np.float32)
    tie = _relu_ties(oracle.sdf_fwd(pts, table, mlp, 64, n_hidden)[2], mlp, 64, n_hidden)
    assert tie.mean() < 2e-2
    v_sdf[tie], v_y1[tie] = 0, 0
    tg, mg, vx = torch.zeros(n_params, device=dev), torch.zeros(len(mlp), device=dev), torch.empty(n, 3, device=dev)
    cabi.sdf_bwd(net, xt, t(v_sdf), t(v_y1), tg, mg, vx, n_variants=variants, delta=delta)
    torch.cuda.synchronize()
    r_tg, r_mg, r_vx = oracle.sdf_bwd(pts, table, mlp, v_sdf, v_y1, 64, n_hidden)
    mgc, tgc, vxc = mg.cpu().numpy(), tg.cpu().numpy(), vx.cpu().numpy()
    assert_close_frac(mgc, r_mg, 1e-4, 3e-5 * np.abs(r_mg).max(), 0.0, "mlp grad (tensor cores)")
    assert np.linalg.norm(mgc - r_mg) <= 5e-5 * np.linalg.norm(r_mg)
    assert_close_frac(tgc, r_tg, 2e-3, 1e-5 * np.abs(r_tg).max(), 1e-3, "table grad (tensor cores)")
    assert np.linalg.norm(tgc - r_tg) <= 2e-4 * np.linalg.norm(r_tg)
    assert_close_frac(vxc, r_vx[:n], 2e-3, 1e-4 * np.abs(r_vx).max(), 1e-3, "v_x (tensor cores)")
    assert np.linalg.norm(vxc - r_vx[:n]) <= 5e-4 * np.linalg.norm(r_vx[:n])


@pytest.mark.parametrize("case", ["ray", "splat", "single"])
def test_sdf_train_fused_equals_separate_calls(oracle, case):
    """gssdf_sdf_train (forward + losses + backward in ONE tensor-core kernel) == gssdf_sdf_fwd + gssdf_sdf_loss + gssdf_sdf_bwd
    (mlp_mode 1) on the two shapes of the training step: ray samples (BCE + eikonal) and splat samples (coupling + eikonal,
    visibility gate, device-side live count, dL/dx)."""
    from gssdf_b200 import cabi
    dev = _dev()
    n, n_hidden = (3000, 3)
    V = 1 if case == "single" else 7
    rng = np.random.default_rng(99)
    n_params, _ = oracle.grid_setup()
    table = rng.uniform(-0.5, 0.5, n_params).astype(np.float32)
    mlp = _mlp(rng, 64, n_hidden)
    x = rng.uniform(0.05, 0.95, (n, 3)).astype(np.float32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    tab, half, mlp_t, xt = t(table), torch.empty(n_params, dtype=torch.float16, device=dev), t(mlp), t(x)
    cabi.sdf_table_to_half(tab, half)
    net = _tc_net(cabi, half, mlp_t, n_hidden)
    delta = 0.01
    gt = t(rng.uniform(-0.1, 0.1, n).astype(np.float32)) if case != "splat" else None
    w = t(rng.uniform(0, 1, (n, 1)).astype(np.float32)) if case == "splat" else None
    vis = t(rng.uniform(0, 1, (n, 1)).astype(np.float32)) if case == "splat" else None
    n_live = torch.tensor([2500, 0, 0, 0], dtype=torch.int32, device=dev) if case == "splat" else None
    kw = dict(visibilities=vis, visible_thr=0.3, n_live=n_live)
    bce_w, eik_w, gs_w, isg = (0.0 if case == "splat" else 1.0), 0.1, (0.5 if case == "splat" else 0.0), 10.0
    # separate calls
    sdf, y1 = torch.zeros(V * n, device=dev), torch.zeros(V * n, device=dev)
    vs, vy = torch.zeros(V * n, device=dev), torch.zeros(V * n, device=dev)
    loss_a = torch.zeros(1, device=dev)
    tg_a, mg_a, vx_a = torch.zeros(n_params, device=dev), torch.zeros(len(mlp), device=dev), torch.zeros(n, 3, device=dev)
    cabi.sdf_fwd(net, xt, sdf, y1, None, n_variants=V, delta=delta, n_live=n_live)
    cabi.sdf_loss(n, V, sdf, y1, gt, w, isg, bce_w, eik_w, gs_w, delta, loss_a, vs, vy, **kw)
    cabi.sdf_bwd(net, xt, vs, vy, tg_a, mg_a, vx_a, n_variants=V, delta=delta, n_live=n_live)
    # fused
    loss_b = torch.zeros(1, device=dev)
    tg_b, mg_b, vx_b = torch.zeros(n_params, device=dev), torch.zeros(len(mlp), device=dev), torch.zeros(n, 3, device=dev)
    cabi.sdf_train(net, xt, V, delta, gt, w, isg, bce_w, eik_w, gs_w, loss_b, tg_b, mg_b, vx_b, **kw)
    torch.cuda.synchronize()
    assert float(loss_a) != 0.0
    assert abs(float(loss_a) - float(loss_b)) <= 1e-5 * abs(float(loss_a))
    for name, a_, b_ in (("mlp grad", mg_a, mg_b), ("table grad", tg_a, tg_b), ("v_x", vx_a, vx_b)):
        a_, b_ = a_.cpu().numpy().astype(np.float64), b_.cpu().numpy().astype(np.float64)
        assert np.abs(a_).max() > 0, name
        # the cotangent reaching the encoding is rounded to fp16 (x128) in both paths; with mean-normalised losses it sits in the
        # fp16 subnormal range, where a 1-ulp difference of the fp32 seeds (different summation order of the 64 -> 2 output
        # layer) flips whole quanta -> table grad / v_x agree at the 1e-3 level only (same effect as in test_sdf_variants_and_losses)
        tol = 2e-5 if name == "mlp grad" else 2e-3
        assert np.linalg.norm(a_ - b_) <= tol * np.linalg.norm(a_), f"{name}: {np.linalg.norm(a_ - b_) / np.linalg.norm(a_):.2e}"


def test_full_step_tensor_core_equals_cuda_core_path():
    """GsSdfStep ([A] SDF on rays, [B] render, [C] GS<->SDF coupling, [D] backward) with the fused tensor-core SDF kernels (mlp_mode 1)
    vs the three-call fp32 CUDA-core path (mlp_mode 0): losses and every segment of the flat gradient agree."""
    import math
    from gssdf_b200 import render, scene as S
    dev = _dev()
    N, W, H, deg = 3000, 160, 96, 2
    sc = S.box_scene(N, deg, seed=0, scale_mult=6.0)
    V, K = S.cameras([0], W, H)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    tsc = {k: t(v) for k, v in sc.items()}
    cfg = dict(n_levels=16, n_features=2, log2_hashmap_size=19, base_resolution=32, per_level_scale=2.0, hidden_dim=64, n_hidden=3)
    gen = torch.Generator(dev).manual_seed(5)
    n_ray = 4096
    outs = []
    for mode in (0, 1):
        G = render.GsSdfStep(N, (deg + 1) ** 2, W, H, dev, 300000, cfg, n_ray_samples=n_ray, sh_degree=deg, map_size=14.0, mlp_mode=mode,
                             eikonal_mode=0)
        gen.manual_seed(5)
        table = (torch.rand(G.n_table, device=dev, generator=gen) * 2 - 1) * 0.1
        chunks, dims = [], [32, 64, 64, 64, 64, 2]
        for k_, o_ in zip(dims[:-1], dims[1:]):
            b_ = 1.0 / math.sqrt(k_)
            chunks += [(torch.rand(o_ * k_, device=dev, generator=gen) * 2 - 1) * b_, (torch.rand(o_, device=dev, generator=gen) * 2 - 1) * b_]
        mlp = torch.cat(chunks)
        box = torch.tensor(S.BOX, device=dev, dtype=torch.float32)
        ray_xyz = (torch.rand(n_ray, 3, device=dev, generator=gen) * 2 - 1) * (box + 0.3)
        ray_gt = (box - ray_xyz.abs()).min(dim=1).values.clamp(-0.3, 0.3).contiguous()
        gt = torch.rand(1, H, W, 4, device=dev, generator=gen)
        loss, sdf_loss = G.step(tsc, table, mlp, t(V), t(K), gt, ray_xyz, ray_gt, t(S.randns(N)))
        torch.cuda.synchronize()
        n_splat = G.R.flat_grad.numel()
        outs.append(dict(loss=float(loss[0]), sdf_loss=float(sdf_loss[0]), splat=G.R.flat_grad.clone(), table=G.table_grad.clone(),
                         mlp=G.mlp_grad.clone(), nnz=G.R.read_counts()["nnz"]))
    a, b = outs
    assert a["nnz"] == b["nnz"] and a["nnz"] > 100
    assert abs(a["loss"] - b["loss"]) <= 1e-5 * abs(a["loss"])
    assert abs(a["sdf_loss"] - b["sdf_loss"]) <= 1e-4 * abs(a["sdf_loss"]) and a["sdf_loss"] != 0.0
    for k, tol in (("mlp", 1e-4), ("table", 3e-3), ("splat", 1e-3)):
        x, y = a[k].double(), b[k].double()
        assert float(x.abs().max()) > 0
        rel = float((x - y).norm() / x.norm())
        assert rel <= tol, f"{k}: {rel:.2e}"


@pytest.mark.parametrize("align_w,n", [(0.1, 1500), (0.0, 1500)])
def test_sdf_train_analytic_eikonal_double_backward(oracle, align_w, n):
    """eikonal_mode 1 (the reference default): eikonal + align losses on the ANALYTIC gradient d sdf/dx and their double backward
    to decoder / table, against the oracle chain (pinned to torch.autograd in tests/test_sdf_oracle.py) with tcnn's fp16
    rounding points (dL/dy -> half x128, half corner products, half dL_ddLdy), at the 1e-3 of DESIGN section 9; and the split
    arrangement of the training step (skip-base 7-variant forward, then V = 1 with sdf_variants) against the V = 7 call."""
    from gssdf_b200 import cabi
    dev = _dev()
    n_hidden, V, delta = 3, 7, 0.01
    rng = np.random.default_rng(31)
    n_params, _ = oracle.grid_setup()
    table = rng.uniform(-2e-3, 2e-3, n_params).astype(np.float32)
    mlp = _mlp(rng, 64, n_hidden)
    # points off the knife edges of the comparison (a hidden pre-activation within 1e-4 of zero, an align-loss sign within 2e-3 |g|):
    # there fp32-grade differences may legitimately flip a discrete choice, so they are left out rather than allowed for by a loose bound
    P = SO.clean_points(oracle, rng, n, table, mlp, n_hidden, (0.5, 0.5, 0.5), 0.0, delta, 0.45)
    x = P["xw"]
    gt = rng.uniform(-0.1, 0.1, n).astype(np.float32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    tab, half, mlp_t, xt = t(table), torch.empty(n_params, dtype=torch.float16, device=dev), t(mlp), t(x)
    cabi.sdf_table_to_half(tab, half)
    net = _tc_net(cabi, half, mlp_t, n_hidden)
    isg, bce_w, eik_w = 10.0, 1.0, 0.1
    # ---- oracle (tests/sdf_train_oracle.py: the oracle chains composed as the kernel composes them)
    R = SO.compose(oracle, P, table, mlp, n_hidden, 0.0, delta, eik_w, align_w, n, gt=gt, bce_isigma=isg, bce_weight=bce_w)
    l1, l2, mg1, mg2, tg1, tg2 = R["loss1"], R["loss2"], R["mlp1"], R["mlp2"], R["table1"], R["table2"]
    # ---- GPU
    loss = torch.zeros(1, device=dev)
    tg, mg = torch.zeros(n_params, device=dev), torch.zeros(len(mlp), device=dev)
    cabi.sdf_train(net, xt, V, delta, t(gt), None, isg, bce_w, eik_w, 0.0, loss, tg, mg, None, eikonal_mode=1, align_weight=align_w)
    # the split arrangement of the training step: forward-only pass over the 7 variants, then the fused kernel on the base points
    loss_s = torch.zeros(1, device=dev)
    tg_s, mg_s, sdf7 = torch.zeros(n_params, device=dev), torch.zeros(len(mlp), device=dev), torch.empty(7 * n, device=dev)
    cabi.sdf_fwd(net, xt, sdf7, None, None, n_variants=7, delta=delta)
    cabi.sdf_train(net, xt, 1, delta, t(gt), None, isg, bce_w, eik_w, 0.0, loss_s, tg_s, mg_s, None, eikonal_mode=1, align_weight=align_w,
                   sdf_variants=sdf7 if align_w > 0 else None)
    torch.cuda.synchronize()
    assert abs(float(loss_s) - float(loss)) <= 1e-5 * abs(float(loss))
    assert float((mg_s - mg).norm()) <= 1e-4 * float(mg.norm()) and float((tg_s - tg).norm()) <= 2e-3 * float(tg.norm())
    assert abs(float(loss) - (l1 + l2)) <= 1e-4 * abs(l1 + l2), (float(loss), l1, l2)
    r_mg, r_tg = mg1 + mg2, tg1 + tg2
    mgc, tgc = mg.cpu().numpy().astype(np.float64), tg.cpu().numpy().astype(np.float64)
    assert np.linalg.norm(mg2) > 1e-3 * np.linalg.norm(mg1)  # the second-order part is a visible share of the reference gradient
    e_m, e_t = np.linalg.norm(mgc - r_mg) / np.linalg.norm(r_mg), np.linalg.norm(tgc - r_tg) / np.linalg.norm(r_tg)
    # the second-order share alone (first-order part removed with the oracle's value)
    e_m2 = np.linalg.norm((mgc - mg1) - mg2) / np.linalg.norm(mg2)
    e_t2 = np.linalg.norm((tgc - tg1) - tg2) / np.linalg.norm(tg2)
    print(f"analytic eikonal, align {align_w}: mlp {e_m:.1e} (2nd {e_m2:.1e}), table {e_t:.1e} (2nd {e_t2:.1e})")
    assert e_m <= 1e-3, f"mlp grad {e_m:.2e}"
    assert e_t <= 1e-3, f"table grad {e_t:.2e}"
    assert e_m2 <= 1e-3 and e_t2 <= 1e-3, (e_m2, e_t2)


@pytest.mark.parametrize("n,live", [(1, None), (19, None), (130, 70), (300, 0)])
def test_sdf_train_small_and_ragged_batches(oracle, n, live):
    """Edge cases of the fused kernel: fewer points than one tile, a partial last tile, a device-side live count below n (and zero):
    analytic and numerical modes must agree with the separate forward / loss / backward calls and leave dead rows alone."""
    from gssdf_b200 import cabi
    dev = _dev()
    rng = np.random.default_rng(n)
    n_params, _ = oracle.grid_setup()
    # tcnn-like amplitudes: with a large table the analytic gradient reaches 1e3..1e4 and the second-order cotangent overflows the
    # binding's fp16 (x128) intermediates to inf / NaN -- in the reference as well (config/base.yaml:12 warns about it)
    table = rng.uniform(-2e-4, 2e-4, n_params).astype(np.float32)
    mlp = _mlp(rng, 64, 3)
    x = rng.uniform(0.05, 0.95, (n, 3)).astype(np.float32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    half, mlp_t, xt = torch.empty(n_params, dtype=torch.float16, device=dev), t(mlp), t(x)
    cabi.sdf_table_to_half(t(table), half)
    net = _tc_net(cabi, half, mlp_t, 3)
    gt = t(rng.uniform(-0.1, 0.1, n).astype(np.float32))
    n_live = torch.tensor([live, 0, 0, 0], dtype=torch.int32, device=dev) if live is not None else None
    delta = 0.01
    # numerical mode vs the three separate calls
    sdf, y1 = torch.zeros(7 * n, device=dev), torch.zeros(7 * n, device=dev)
    vs, vy = torch.zeros(7 * n, device=dev), torch.zeros(7 * n, device=dev)
    la, tga, mga = torch.zeros(1, device=dev), torch.zeros(n_params, device=dev), torch.zeros(len(mlp), device=dev)
    cabi.sdf_fwd(net, xt, sdf, y1, None, n_variants=7, delta=delta, n_live=n_live)
    cabi.sdf_loss(n, 7, sdf, y1, gt, None, 10.0, 1.0, 0.1, 0.0, delta, la, vs, vy, n_live=n_live)
    cabi.sdf_bwd(net, xt, vs, vy, tga, mga, None, n_variants=7, delta=delta, n_live=n_live)
    lb, tgb, mgb = torch.zeros(1, device=dev), torch.zeros(n_params, device=dev), torch.zeros(len(mlp), device=dev)
    vx = torch.full((n, 3), 7.0, device=dev)
    cabi.sdf_train(net, xt, 7, delta, gt, None, 10.0, 1.0, 0.1, 0.0, lb, tgb, mgb, vx, n_live=n_live)
    # analytic mode, both arrangements
    lc, tgc, mgc = torch.zeros(1, device=dev), torch.zeros(n_params, device=dev), torch.zeros(len(mlp), device=dev)
    cabi.sdf_train(net, xt, 7, delta, gt, None, 10.0, 1.0, 0.1, 0.0, lc, tgc, mgc, None, n_live=n_live, eikonal_mode=1, align_weight=0.1)
    ld, tgd, mgd = torch.zeros(1, device=dev), torch.zeros(n_params, device=dev), torch.zeros(len(mlp), device=dev)
    cabi.sdf_fwd(net, xt, sdf, None, None, n_variants=7, delta=delta, n_live=n_live, skip_base_variant=True)
    cabi.sdf_train(net, xt, 1, delta, gt, None, 10.0, 1.0, 0.1, 0.0, ld, tgd, mgd, None, n_live=n_live, eikonal_mode=1, align_weight=0.1,
                   sdf_variants=sdf)
    torch.cuda.synchronize()
    nl = n if live is None else live
    if nl == 0:
        for z in (la, lb, lc, ld, mgb, mgc, mgd, tgb, tgc, tgd):
            assert float(z.abs().sum()) == 0.0
        assert float((vx - 7.0).abs().sum()) == 0.0
        return
    assert abs(float(la) - float(lb)) <= 1e-5 * abs(float(la))
    assert float((mga - mgb).norm()) <= 1e-4 * float(mga.norm())
    # (table gradients of tiny batches sit in the fp16 subnormal range of the binding's x128 cotangent: quantum-level agreement only)
    assert float((tga - tgb).norm()) <= 2e-2 * float(tga.norm())
    assert float((vx[nl:] - 7.0).abs().sum()) == 0.0 and bool(torch.isfinite(vx[:nl]).all())
    assert abs(float(lc) - float(ld)) <= 1e-5 * abs(float(lc)) and np.isfinite(float(lc))
    assert bool(torch.isfinite(tgc).all()) and bool(torch.isfinite(mgc).all())
    assert float((mgc - mgd).norm()) <= 1e-4 * float(mgc.norm()) and float((tgc - tgd).norm()) <= 2e-2 * float(tgc.norm())


def test_cuda_features_match_tiny_cuda_nn_kernels(oracle):
    """The CUDA encoder against the outputs of tiny-cuda-nn's own kernel_grid run on an H100 (tests/golden/tcnn_grid_ref.npz; level 0
    dense incl. cube-face points, levels 1-15 hashed at log2_hashmap_size 16): bit-identical features, both arithmetic modes."""
    import os
    from gssdf_b200 import cabi
    dev = _dev()
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tcnn_grid_ref.npz"))
    rng = np.random.default_rng(int(g["seed"]))
    table = rng.uniform(-0.5, 0.5, int(g["n_params"])).astype(np.float32)
    n = g["x"].shape[0]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    half, mlp_t, xt = torch.empty(len(table), dtype=torch.float16, device=dev), t(_mlp(np.random.default_rng(1), 64, 3)), t(g["x"])
    cabi.sdf_table_to_half(t(table), half)
    for mode in (0, 1):
        net = cabi.sdf_net(half, mlp_t, log2_hashmap_size=int(g["cfg"][1]), hidden_dim=64, n_hidden=3)
        if mode == 1:
            packed = torch.empty(cabi.sdf_mlp_packed_bytes(net), dtype=torch.uint8, device=dev)
            cabi.sdf_mlp_pack(net, packed)
            _KEEP.append(packed)
            net = cabi.sdf_net(half, mlp_t, log2_hashmap_size=int(g["cfg"][1]), hidden_dim=64, n_hidden=3, mlp_mode=1, mlp_packed=packed)
        assert cabi.sdf_table_params(net) == len(table)
        sdf, feat = torch.empty(n, device=dev), torch.empty(n, 32, device=dev)
        cabi.sdf_fwd(net, xt, sdf, None, feat)
        torch.cuda.synchronize()
        assert np.array_equal(feat.cpu().numpy(), g["enc"]), f"mlp_mode {mode}"
