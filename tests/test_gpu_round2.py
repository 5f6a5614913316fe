"""Round-2 GPU parity: operator-level hash grid (fwd / bwd / bwd-bwd) vs the oracle and tiny-cuda-nn's own kernels, the tcnn_binding
twin (TCNNEncoding through libtorch autograd incl. double backward) replaying the reference's LocalMap call sequences, the fused Adam,
the normal-consistency and isotropic losses, the coupling-site sample gate, non-default CUDA streams, and the analytic eikonal at 1e-3."""
import json
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _mlp(rng, hidden, n_hidden, in_dim=32):
    dims = [in_dim] + [hidden] * (1 + n_hidden) + [2]
    ps = []
    for k, o in zip(dims[:-1], dims[1:]):
        b = 1 / np.sqrt(k)
        ps += [rng.uniform(-b, b, o * k), rng.uniform(-b, b, o)]
    return np.concatenate(ps).astype(np.float32)


def _min_preact(oracle, x01, table, mlp, hidden, n_hidden):
    """smallest |hidden pre-activation| of every point (fp64 decoder on the oracle's features)."""
    feat = oracle.hashgrid_fwd(x01, table)
    a, o, K = feat.astype(np.float64), 0, feat.shape[1]
    m = np.full(len(feat), np.inf)
    for _ in range(1 + n_hidden):
        W = mlp[o:o + hidden * K].reshape(hidden, K).astype(np.float64)
        b = mlp[o + hidden * K:o + hidden * K + hidden].astype(np.float64)
        o += hidden * K + hidden
        z = a @ W.T + b
        m = np.minimum(m, np.abs(z).min(1))
        a, K = np.maximum(z, 0), hidden
    return m


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


# ------------------------------------------------------------------------------------------------------------------------------
def test_ops_honour_the_current_stream():
    """ADVICE r1: the ctypes binding passed the 64-bit cudaStream_t as a C int. With typed argtypes an op launched under
    torch.cuda.stream(side) must run on `side` (ordered after work queued there) and give the default-stream result."""
    from gssdf_b200 import cabi
    dev = _dev()
    n = 1 << 20
    src = torch.randn(n, device=dev)
    ref = torch.empty(n, dtype=torch.float16, device=dev)
    cabi.sdf_table_to_half(src, ref)
    torch.cuda.synchronize()
    side = torch.cuda.Stream(device=dev)
    assert side.cuda_stream > 0xFFFFFFFF or side.cuda_stream != 0
    out = torch.zeros(n, dtype=torch.float16, device=dev)
    src2 = torch.empty(n, device=dev)
    with torch.cuda.stream(side):
        torch.cuda._sleep(20_000_000)  # keeps `side` busy: a launch on the wrong (default) stream would read src2 before the copy below
        src2.copy_(src)
        cabi.sdf_table_to_half(src2, out)
    side.synchronize()
    assert torch.equal(out, ref)


# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("log2", [19, 16])
def test_hashgrid_operators_vs_oracle(oracle, log2):
    from gssdf_b200 import cabi
    dev = _dev()
    rng = np.random.default_rng(log2)
    cfg = dict(L=16, F=2, log2_hashmap=log2, base_res=32, per_level_scale=2.0)
    n_params, _ = oracle.grid_setup(**cfg)
    table = rng.uniform(-0.5, 0.5, n_params).astype(np.float32)
    n = 3000
    x = rng.uniform(0.02, 0.98, (n, 3)).astype(np.float32)
    x[:32] = rng.choice(np.array([0.0, 1.0, 0.99, 0.985], np.float32), (32, 3))
    gy = (rng.standard_normal((n, 32)) * 0.05).astype(np.float32)
    cc = (rng.standard_normal((n, 3)) * 1e-3).astype(np.float32)
    half = torch.empty(n_params, dtype=torch.float16, device=dev)
    cabi.sdf_table_to_half(_t(table, dev), half)
    net = cabi.sdf_net(half, None, log2_hashmap_size=log2)
    xt = _t(x, dev)
    feat = torch.empty(n, 32, device=dev)
    cabi.hashgrid_fwd(net, xt, feat)
    r_feat, dy = oracle.hashgrid_fwd(x, table, want_dy_dx=True, **cfg)
    assert np.array_equal(feat.cpu().numpy(), r_feat), "features must be bit-identical"
    tg, dx = torch.zeros(n_params, device=dev), torch.empty(n, 3, device=dev)
    cabi.hashgrid_bwd(net, xt, _t(gy, dev), tg, dx)
    r_tg, r_dx = oracle.hashgrid_bwd(x, gy, n_params, dy, **cfg)
    assert rel(tg.cpu().numpy(), r_tg) <= 1e-5
    assert rel(dx.cpu().numpy(), r_dx) <= 1e-5
    tg2, ddy, dx2 = torch.zeros(n_params, device=dev), torch.empty(n, 32, device=dev), torch.empty(n, 3, device=dev)
    cabi.hashgrid_bwdbwd(net, xt, _t(cc, dev), _t(gy, dev), tg2, ddy, dx2)
    r_tg2, r_ddy = oracle.hashgrid_bwd_bwd(x, cc, gy, n_params, dy, **cfg)
    r_dx2 = oracle.hashgrid_bwd_bwd_input(x, cc, gy, table, **cfg)
    assert rel(tg2.cpu().numpy(), r_tg2) <= 1e-5
    d = ddy.cpu().numpy()
    # fp32 sum order of the three dy_dx * cc products: half an fp16 ulp (2^-11 relative) on isolated entries, more only where the three
    # terms cancel (absolute floor relative to the row's largest entry)
    assert (d != r_ddy).mean() <= 2e-3
    assert (np.abs(d - r_ddy) <= 2e-3 * np.abs(r_ddy) + 2e-3 * np.abs(r_ddy).max(1, keepdims=True)).all() and rel(d, r_ddy) <= 1e-3
    assert rel(dx2.cpu().numpy(), r_dx2) <= 1e-4, rel(dx2.cpu().numpy(), r_dx2)
    # NULL outputs / empty batch are legal
    cabi.hashgrid_bwd(net, xt, _t(gy, dev), None, dx)
    cabi.hashgrid_bwdbwd(net, xt, _t(cc, dev), _t(gy, dev), None, ddy, None)
    cabi.hashgrid_fwd(net, xt[:0], feat[:0])


@pytest.mark.parametrize("name", ["tcnn_grid_ref.npz", "tcnn_grid_ref19.npz"])
def test_hashgrid_operators_vs_tiny_cuda_nn_goldens(name):
    """Our operator-level kernels fed with the SAME inputs as tiny-cuda-nn's own kernels (goldens from oracle/gen_golden_tcnn.py run on a
    H100): kernel_grid, kernel_grid_backward(+_input), kernel_grid_backward_input_backward_{grid,dLdoutput,input}."""
    from gssdf_b200 import cabi
    path = os.path.join(HERE, "golden", name)
    if not os.path.exists(path):
        pytest.skip(name + " not generated yet")
    dev = _dev()
    g = np.load(path)
    rng = np.random.default_rng(int(g["seed"]))
    n_params, log2 = int(g["n_params"]), int(g["cfg"][1])
    table = rng.uniform(-0.5, 0.5, n_params).astype(np.float32)
    half = torch.empty(n_params, dtype=torch.float16, device=dev)
    cabi.sdf_table_to_half(_t(table, dev), half)
    net = cabi.sdf_net(half, None, log2_hashmap_size=log2)
    x, n = g["x"], len(g["x"])
    xt = _t(x, dev)
    feat = torch.empty(n, 32, device=dev)
    cabi.hashgrid_fwd(net, xt, feat)
    assert np.array_equal(feat.cpu().numpy(), g["enc"])
    tg, dx = torch.zeros(n_params, device=dev), torch.empty(n, 3, device=dev)
    cabi.hashgrid_bwd(net, xt, _t(g["dL_dy"], dev), tg, dx)
    ref_tg = np.zeros(n_params)
    ref_tg[g["grid_grad_idx"]] = g["grid_grad_val"].astype(np.float64) / 128.0
    assert rel(tg.cpu().numpy(), ref_tg) <= 2e-3  # the reference accumulates with fp16 atomics (a rounding per add)
    assert np.allclose(dx.cpu().numpy(), g["dL_dx_scaled"] / 128.0, rtol=2e-5, atol=1e-6 * np.abs(g["dL_dx_scaled"]).max() / 128.0)
    tg2, ddy, dx2 = torch.zeros(n_params, device=dev), torch.empty(n, 32, device=dev), torch.empty(n, 3, device=dev)
    cabi.hashgrid_bwdbwd(net, xt, _t(g["cc"], dev), _t(g["dL_dy"], dev), tg2, ddy, dx2)
    t2 = tg2.cpu().numpy().astype(np.float64)
    ref_tg2 = np.zeros(n_params)
    ref_tg2[g["grid_grad2_idx"]] = g["grid_grad2_val"].astype(np.float64) / 128.0
    fin = np.isfinite(ref_tg2) & np.isfinite(t2)
    small = fin & (np.abs(ref_tg2) < 100.0)  # far from the half range limit of the reference's fp16 accumulator (65504 / 128)
    assert small.mean() > 0.99 or name == "tcnn_grid_ref.npz"
    assert rel(t2[small], ref_tg2[small]) <= 2e-3
    d = ddy.cpu().numpy()
    okd = np.isfinite(g["dL_ddLdy"])
    assert np.allclose(d[okd], g["dL_ddLdy"][okd], rtol=2e-3, atol=0)
    if "dL_dx2_scaled" in g:
        r = g["dL_dx2_scaled"].astype(np.float64) / 128.0
        ok = np.isfinite(r).all(1)
        e = rel(dx2.cpu().numpy()[ok], r[ok])
        print(f"{name}: input double backward vs tcnn: rel L2 {e:.2e}")
        assert e <= 1e-4, e


# ------------------------------------------------------------------------------------------------------------------------------
def test_tcnn_binding_twin_replays_local_map(oracle):
    """shim/include/tcnn_binding/tcnn_binding.h through libtorch autograd, driven by a C++ replay of the reference's call sequences
    (EncodingMap ctor / encoding, LocalMap ctor / get_sdf / get_gradient analytic with create_graph, sdf_regularization; statements
    copied in meaning from encoding_map.cpp:15-26,31-60, local_map.cpp:26-42,73-75,87-103,150-171, neural_mapping.cpp:106-136):
    values and every gradient (encoder parameters incl. the double backward, decoder) vs the oracle chain and vs the fused kernel."""
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "gs-sdf_b200"))
    from gssdf_b200 import cabi
    try:
        import gssdf_shim
    except ImportError as e:
        pytest.fail(f"gssdf_shim.so missing (python gs-sdf_b200/build.py): {e}")
    dev = _dev()
    rng = np.random.default_rng(77)
    hidden, n_hidden, map_size, bce_sigma, delta = 64, 3, 14.0, 0.1, 0.1
    L = gssdf_shim.LocalMapReplay(16, 2, 19, hidden, n_hidden, map_size, bce_sigma)
    enc = L.encoder_params()
    n_params, _ = oracle.grid_setup()
    assert enc.numel() == n_params and enc.dtype == torch.float32 and enc.requires_grad
    assert float(enc.abs().max()) <= 1e-4 and float(enc.std()) > 4e-5  # U(-1e-4, 1e-4)
    table = rng.uniform(-2e-3, 2e-3, n_params).astype(np.float32)
    mlp = _mlp(rng, hidden, n_hidden)
    with torch.no_grad():
        enc.copy_(_t(table, dev))  # in-place: bumps the version counter -> the fp16 shadow must refresh
    L.set_decoder(_t(mlp, dev))
    # points whose ReLU pattern is stable (|pre-activation| > 1e-4): the double backward is discontinuous across a flip
    xw = rng.uniform(-6.0, 6.0, (6000, 3)).astype(np.float32)
    x01 = (0.5 * (xw * 2.0 * np.float32(1.0 / map_size)) + 0.5).astype(np.float32)
    keep = _min_preact(oracle, x01, table, mlp, hidden, n_hidden) > 1e-4
    xw, x01 = xw[keep][:2048], x01[keep][:2048]
    n = len(xw)
    assert n == 2048
    xt = _t(xw, dev)
    sdf, isigma = L.get_sdf(xt)
    r_sdf, r_y1, _ = oracle.sdf_fwd(x01, table, mlp, hidden, n_hidden)
    assert rel(sdf.detach().cpu().numpy()[:, 0], r_sdf) <= 1e-5
    sp = np.where(100 * r_y1 > 20, r_y1, np.log1p(np.exp(np.minimum(100 * r_y1, 20))) / 100)
    assert rel(isigma.detach().cpu().numpy()[:, 0], 1 + sp / bce_sigma) <= 1e-5
    # analytic gradient (world units: d/dx01 * 1/map_size)
    g = L.get_gradient_analytic(xt.clone())
    r_g = oracle.sdf_grad_analytic(x01, table, mlp, hidden, n_hidden).astype(np.float64) / map_size
    e_g = rel(g.detach().cpu().numpy(), r_g)
    # eikonal + align through the double backward
    L.zero_grad()
    loss = L.regularization(xt, delta, 0.1, 0.1)
    loss.backward()
    torch.cuda.synchronize()
    enc_g, dec_g = L.encoder_params().grad.cpu().numpy().astype(np.float64), L.decoder_grad().cpu().numpy().astype(np.float64)
    # oracle chain
    offs = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.float32) * np.float32(delta)
    pts01 = (0.5 * ((xw[None] + offs[:, None]).reshape(-1, 3) * 2.0 * np.float32(1.0 / map_size)) + 0.5).astype(np.float32)
    s6 = oracle.sdf_fwd(pts01, table, mlp, hidden, n_hidden)[0].reshape(6, n).astype(np.float64)
    gnum = np.stack([s6[0] - s6[1], s6[2] - s6[3], s6[4] - s6[5]], 1) * (0.5 / delta)
    nrm = np.linalg.norm(r_g, axis=1)
    r_loss = 0.1 * np.mean((nrm - 1) ** 2) + 0.1 * np.mean(np.abs(r_g - gnum))
    c = (0.1 / n) * (2 * (nrm - 1) / nrm)[:, None] * r_g + (0.1 / (3 * n)) * np.sign(r_g - gnum)
    r_tg, r_mg = oracle.sdf_grad_analytic_bwd(x01, table, mlp, (c / map_size).astype(np.float32), hidden, n_hidden)
    e_l, e_t, e_m = abs(float(loss) - r_loss) / abs(r_loss), rel(enc_g, r_tg), rel(dec_g, r_mg)
    print(f"tcnn twin vs oracle: grad {e_g:.2e} loss {e_l:.2e} table-grad {e_t:.2e} decoder-grad {e_m:.2e}")
    assert e_g <= 1e-4 and e_l <= 1e-4
    assert e_t <= 1e-3 and e_m <= 1e-3
    # ... and vs the fused tensor-core kernel (same losses on the same points)
    half = torch.empty(n_params, dtype=torch.float16, device=dev)
    cabi.sdf_table_to_half(_t(table, dev), half)
    mlp_t = _t(mlp, dev)
    probe = cabi.sdf_net(half, mlp_t)
    packed = torch.empty(cabi.sdf_mlp_packed_bytes(probe), dtype=torch.uint8, device=dev)
    cabi.sdf_mlp_pack(probe, packed)
    net = cabi.sdf_net(half, mlp_t, mlp_mode=1, mlp_packed=packed, inv_size=1.0 / map_size)
    fl, tg, mg = torch.zeros(1, device=dev), torch.zeros(n_params, device=dev), torch.zeros(len(mlp), device=dev)
    cabi.sdf_train(net, xt, 7, delta, None, None, 1.0 / bce_sigma, 0.0, 0.1, 0.0, fl, tg, mg, None, eikonal_mode=1, align_weight=0.1)
    torch.cuda.synchronize()
    f_l, f_t, f_m = abs(float(fl) - float(loss)) / abs(float(loss)), rel(tg.cpu().numpy(), enc_g), rel(mg.cpu().numpy(), dec_g)
    print(f"fused kernel vs tcnn twin: loss {f_l:.2e} table-grad {f_t:.2e} decoder-grad {f_m:.2e}")
    assert f_l <= 1e-4 and f_t <= 1e-3 and f_m <= 1e-3
    # curvature branch of get_gradient (local_map.cpp:161-166): Hessian row sums = a second autograd.grad through the encoding's double
    # backward (kernel_grid_backward_input_backward_input; the ReLU decoder is piecewise linear, so d(d sdf/d feat)/dx = 0 a.e.)
    gh, hh = L.get_gradient_hessian_analytic(xt.clone())
    widths = [32] + [hidden] * (1 + n_hidden) + [2]
    r_feat = oracle.hashgrid_fwd(x01, table)
    d_out = np.zeros((n, 2)); d_out[:, 0] = 1.0
    dfeat, _ = oracle.mlp_bwd(r_feat, widths, mlp, d_out)
    r_h = oracle.hashgrid_bwd_bwd_input(x01, np.ones((n, 3), np.float32), dfeat.astype(np.float32), table).astype(np.float64) / map_size ** 2
    e_h = rel(hh.detach().cpu().numpy(), r_h)
    print(f"tcnn twin: Hessian row sums vs oracle {e_h:.2e}")
    assert rel(gh.detach().cpu().numpy(), r_g) <= 1e-4 and e_h <= 2e-3
    # unsupported configurations fail like tcnn's CHECK_THROW (std::runtime_error)
    with pytest.raises(RuntimeError):
        gssdf_shim.TCNNEncoding(3, json.dumps({"otype": "Grid", "type": "Dense"}), "e", 1337)
    with pytest.raises(RuntimeError):
        gssdf_shim.make_tcnn_network(32, 2, json.dumps({"otype": "FullyFusedMLP"}))


def test_tcnn_encoding_shadow_tracks_optimizer(oracle):
    """params_ stays a flat fp32 parameter; the fp16 shadow follows torch::optim-style in-place updates and set_data / reassignment."""
    import gssdf_shim
    dev = _dev()
    cfg = json.dumps({"otype": "Grid", "type": "Hash", "n_levels": 16, "n_features_per_level": 2, "log2_hashmap_size": 16,
                      "base_resolution": 32, "per_level_scale": 2.0, "interpolation": "Linear"})
    E = gssdf_shim.TCNNEncoding(3, cfg, "enc", 1337)
    assert E.get_out_dim() == 32
    gcfg = dict(L=16, F=2, log2_hashmap=16, base_res=32, per_level_scale=2.0)
    n_params, _ = oracle.grid_setup(**gcfg)
    p = E.params_
    assert p.numel() == n_params
    x = np.random.default_rng(0).uniform(0, 1, (500, 3)).astype(np.float32)
    xt = _t(x, dev)
    for it in range(3):
        f = E.forward(xt)
        assert np.array_equal(f.cpu().numpy(), oracle.hashgrid_fwd(x, p.detach().cpu().numpy(), **gcfg)), it
        with torch.no_grad():
            p.mul_(1.5).add_(1e-5)  # what an optimiser does
    p.requires_grad_(True)
    f = E.forward(xt)
    f.sum().backward()
    r_tg, _ = oracle.hashgrid_bwd(x, np.ones((500, 32), np.float32), n_params, None, **gcfg)
    assert rel(p.grad.cpu().numpy(), r_tg) <= 1e-5


# ------------------------------------------------------------------------------------------------------------------------------
def test_adam_step_matches_torch_adam():
    """gssdf_adam_step vs torch.optim.Adam (fp64, CPU; betas (0.9, 0.999), eps 1e-15, per-group lr): parameters after 4 steps, the zeroed
    gradient, the fp16 shadow of the table group, odd sizes / unaligned group offsets."""
    from gssdf_b200 import cabi
    dev = _dev()
    g = torch.Generator("cpu").manual_seed(4)
    sizes, lrs = [30001, 4099, 7, 20000, 50002], [1.6e-4, 1e-3, 5e-3, 5e-2, 5e-3]
    offs, o = [], 0
    for s_ in sizes:
        offs.append(o)
        o += s_ + (3 if s_ == 7 else 0)  # a gap: groups need not be contiguous
    total = o
    p0 = torch.randn(total, generator=g, dtype=torch.float64)
    params, grads = p0.float().to(dev), torch.zeros(total, device=dev)
    m, v = torch.zeros(total, device=dev), torch.zeros(total, device=dev)
    half = torch.zeros(sizes[4], dtype=torch.float16, device=dev)
    ref = [p0[o_:o_ + s_].clone().requires_grad_(True) for o_, s_ in zip(offs, sizes)]
    opt = torch.optim.Adam([dict(params=[r], lr=lr) for r, lr in zip(ref, lrs)], betas=(0.9, 0.999), eps=1e-15)
    groups = [(o_, s_, lr, i == 4) for i, (o_, s_, lr) in enumerate(zip(offs, sizes, lrs))]
    for step in range(1, 5):
        gr = torch.randn(total, generator=g, dtype=torch.float64) * (10.0 ** torch.randint(-6, 1, (total,), generator=g).double())
        gr[::7] = 0.0  # untouched rows (invisible splats) still move by their momentum
        grads.copy_(gr.float())
        for r, o_, s_ in zip(ref, offs, sizes):
            r.grad = gr[o_:o_ + s_].float().double() * 0.5
        opt.step()
        cabi.adam_step(params, grads, m, v, groups, step, grad_scale=0.5, zero_grads=True, table_half=half)
    torch.cuda.synchronize()
    for o_, s_ in zip(offs, sizes):
        assert float(grads[o_:o_ + s_].abs().max()) == 0.0  # zero_grad fused into the step (group ranges only)
    got = params.cpu().double()
    for r, o_, s_ in zip(ref, offs, sizes):
        e = float((got[o_:o_ + s_] - r.detach()).abs().max() / r.detach().abs().max())
        assert e <= 2e-6, e
    assert torch.equal(got[offs[2] + 7:offs[3]], p0[offs[2] + 7:offs[3]].float().double())  # the gap is untouched
    assert torch.equal(half.cpu(), params[offs[4]:offs[4] + sizes[4]].half().cpu())


# ------------------------------------------------------------------------------------------------------------------------------
def _depth_to_normal_ref(depth, V, K):
    """sensor::depth_to_normal (cameras.hpp:176-226) in torch, in depth's precision (fp64 as the reference arbiter): depth [H,W,1],
    V world->camera [4,4], K [3,3] of the same dtype."""
    H, W = depth.shape[:2]
    ys, xs = torch.meshgrid(torch.arange(H, dtype=depth.dtype), torch.arange(W, dtype=depth.dtype), indexing="ij")
    zdir = torch.stack([(xs + 0.5 - K[0, 2]) / K[0, 0], (ys + 0.5 - K[1, 2]) / K[1, 1], torch.ones_like(xs)], -1)
    rot = V[:3, :3].T  # camera -> world
    pos = -rot @ V[:3, 3]
    pts = (zdir @ rot.T) * depth + pos
    out = torch.zeros_like(pts)
    dx = pts[2:, 1:-1] - pts[:-2, 1:-1]
    dy = pts[1:-1, 2:] - pts[1:-1, :-2]
    out[1:-1, 1:-1] = torch.nn.functional.normalize(torch.cross(dx, dy, dim=-1), dim=-1)
    return out


@pytest.mark.parametrize("W,H", [(160, 96), (37, 21)])
def test_normal_consistency_loss_matches_reference_formula(W, H):
    """neural_mapping.cpp:243-266 restated with torch fp64 autograd vs the fused kernel: loss, dL/d depth, dL/d render_normal."""
    from gssdf_b200 import cabi, scene as S
    dev = _dev()
    g = torch.Generator("cpu").manual_seed(W)
    Vn, Kn = S.camera(3, W, H)
    V, K = torch.from_numpy(Vn).double(), torch.from_numpy(Kn).double()
    depth = (1.0 + torch.rand(H, W, 1, generator=g, dtype=torch.float64) * 2).requires_grad_(True)
    with torch.no_grad():
        depth[5:9, 5:9] = 0.0  # empty pixels: ED = nan_to_num(0/0) = 0 -> degenerate stencils (zero cross product)
    alpha = torch.rand(H, W, 1, generator=g, dtype=torch.float64)
    rn = torch.nn.functional.normalize(torch.randn(H, W, 3, generator=g, dtype=torch.float64), dim=-1).requires_grad_(True)
    w = 0.01
    dn = _depth_to_normal_ref(depth, V, K) * alpha
    ref = w * (alpha.square().squeeze(-1) - (dn * rn).sum(-1).nan_to_num()).mean()
    ref.backward()
    out_colors = torch.zeros(1, H, W, 4, device=dev)
    out_colors[0, ..., 3] = depth.detach().float().squeeze(-1).to(dev)
    v_out = torch.full((1, H, W, 4), 0.25, device=dev)
    v_n = torch.full((1, H, W, 3), 9.0, device=dev)
    loss = torch.zeros(1, device=dev)
    cabi.normal_consistency_loss(1, W, H, _t(Vn[None], dev), _t(Kn[None], dev), out_colors.data_ptr() + 12, 4,
                                 alpha.float().to(dev).contiguous().view(1, H, W, 1), rn.detach().float().to(dev).contiguous().view(1, H, W, 3),
                                 w, loss, v_depth=v_out.data_ptr() + 12, v_depth_stride=4, v_out_normals=v_n)
    torch.cuda.synchronize()
    assert abs(float(loss) - float(ref)) <= 1e-5 * abs(float(ref))
    assert float((v_out[..., :3] - 0.25).abs().max()) == 0.0
    gd = (v_out[0, ..., 3] - 0.25).cpu().double()
    assert float((gd - depth.grad.squeeze(-1)).abs().max()) <= 1e-4 * float(depth.grad.abs().max()), \
        float((gd - depth.grad.squeeze(-1)).abs().max() / depth.grad.abs().max())
    assert float((v_n[0].cpu().double() - rn.grad).abs().max()) <= 1e-5 * float(rn.grad.abs().max())


def test_isotropic_loss_matches_reference_formula():
    from gssdf_b200 import cabi
    dev = _dev()
    g = torch.Generator("cpu").manual_seed(1)
    N, nnz = 5000, 1800
    raw = (torch.randn(N, 3, generator=g, dtype=torch.float64) * 0.5 - 3).requires_grad_(True)
    gid = torch.randperm(N, generator=g)[:nnz].sort().values
    scale = torch.exp(raw).index_select(0, gid)[:, :2]
    ref = 0.05 * (scale - scale.mean(-1, True)).abs().mean()
    ref.backward()
    counts = cabi.new_counts(dev, nnz=nnz)
    gids = torch.zeros(N, dtype=torch.int64, device=dev)
    gids[:nnz] = gid.to(dev)
    loss, v = torch.zeros(1, device=dev), torch.zeros(N, 3, device=dev)
    cabi.isotropic_loss(N, N, counts, gids, raw.detach().float().to(dev), True, 0.05, loss, v)
    torch.cuda.synchronize()
    assert abs(float(loss) - float(ref)) <= 1e-5 * float(ref)
    assert float((v.cpu().double() - raw.grad).abs().max()) <= 1e-5 * float(raw.grad.abs().max())


# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["numerical", "analytic"])
def test_coupling_site_sample_gate(oracle, mode):
    """ADVICE r1 / neural_mapping.cpp:428-452: with a mixed-visibility (and partly invalid) batch, eikonal / align / coupling act on the
    samples with `valid & vis > thr` only and the means divide by that count: the gated call on all n samples must equal the ungated
    call on the selected subset."""
    from gssdf_b200 import cabi
    dev = _dev()
    rng = np.random.default_rng(9)
    n, delta, thr = 900, 0.01, 0.1
    n_params, _ = oracle.grid_setup()
    table = rng.uniform(-2e-4, 2e-4, n_params).astype(np.float32)
    mlp = _mlp(rng, 64, 3)
    x = rng.uniform(0.05, 0.95, (n, 3)).astype(np.float32)
    vis = rng.uniform(0, 0.3, n).astype(np.float32)
    valid = (rng.uniform(0, 1, n) > 0.2).astype(np.uint8)
    w = rng.uniform(0.2, 1.0, n).astype(np.float32)
    sel = (vis > thr) & (valid != 0)
    assert 100 < sel.sum() < n - 100
    half, mlp_t = torch.empty(n_params, dtype=torch.float16, device=dev), _t(mlp, dev)
    cabi.sdf_table_to_half(_t(table, dev), half)
    probe = cabi.sdf_net(half, mlp_t)
    packed = torch.empty(cabi.sdf_mlp_packed_bytes(probe), dtype=torch.uint8, device=dev)
    cabi.sdf_mlp_pack(probe, packed)
    net = cabi.sdf_net(half, mlp_t, mlp_mode=1, mlp_packed=packed)
    kw = dict(eikonal_mode=1, align_weight=0.1) if mode == "analytic" else {}

    def run(xs, ws, vs, gate):
        m = len(xs)
        loss, tg, mg, vx = torch.zeros(1, device=dev), torch.zeros(n_params, device=dev), torch.zeros(len(mlp), device=dev), torch.zeros(m, 3, device=dev)
        g = {}
        if gate:
            ng = torch.zeros(1, dtype=torch.int32, device=dev)
            vm = _t(valid, dev)
            cabi.sdf_gate_count(m, ng, visibilities=vs, visible_thr=thr, valid_mask=vm)
            assert int(ng) == int(sel.sum())
            g = dict(valid_mask=vm, n_gate=ng)
        cabi.sdf_train(net, xs, 7, delta, None, ws, 10.0, 0.0, 0.1, 1e-3, loss, tg, mg, vx, visibilities=vs, visible_thr=thr, **kw, **g)
        torch.cuda.synchronize()
        return float(loss), tg.cpu().numpy(), mg.cpu().numpy(), vx.cpu().numpy()

    la, tga, mga, vxa = run(_t(x, dev), _t(w, dev), _t(vis, dev), True)
    lb, tgb, mgb, vxb = run(_t(x[sel], dev), _t(w[sel], dev), _t(vis[sel], dev), False)
    assert abs(la - lb) <= 1e-5 * abs(lb) and lb != 0.0
    # (same arithmetic per point; the points sit in different tiles, so the fp32 accumulation order of the sums differs)
    assert rel(mga, mgb) <= 1e-4 and rel(tga, tgb) <= 1e-4
    assert np.abs(vxa[~sel]).max() == 0.0 and rel(vxa[sel], vxb) <= 1e-4
    if mode == "numerical":  # the three-call path (sdf_loss) applies the same gate
        sdf, y1 = torch.zeros(7 * n, device=dev), torch.zeros(7 * n, device=dev)
        vs_, vy_, l3 = torch.zeros(7 * n, device=dev), torch.zeros(7 * n, device=dev), torch.zeros(1, device=dev)
        ng = torch.zeros(1, dtype=torch.int32, device=dev)
        vm = _t(valid, dev)
        cabi.sdf_gate_count(n, ng, visibilities=_t(vis, dev), visible_thr=thr, valid_mask=vm)
        cabi.sdf_fwd(net, _t(x, dev), sdf, y1, None, n_variants=7, delta=delta)
        cabi.sdf_loss(n, 7, sdf, y1, None, _t(w, dev), 10.0, 0.0, 0.1, 1e-3, delta, l3, vs_, vy_, visibilities=_t(vis, dev), visible_thr=thr,
                      valid_mask=vm, n_gate=ng)
        torch.cuda.synchronize()
        assert abs(float(l3) - la) <= 1e-5 * abs(la)
        assert float(vs_.view(7, n)[:, _t(~sel, dev)].abs().max()) == 0.0


# ------------------------------------------------------------------------------------------------------------------------------
def test_analytic_eikonal_double_backward_1e3(oracle):
    """VERDICT r1 weak #1: the reference-default mode at <= 1e-3 (was 2e-2 / 5e-2). Points whose ReLU pattern is unstable (a hidden
    pre-activation within 1e-4 of zero: the double backward is discontinuous there, and fp32 / fp64 evaluations may legitimately land
    on different sides) are excluded from the batch instead of being allowed for by a loose tolerance."""
    from gssdf_b200 import cabi
    dev = _dev()
    rng = np.random.default_rng(31)
    n_hidden, delta, isg, bce_w, eik_w, align_w = 3, 0.01, 10.0, 1.0, 0.1, 0.1
    n_params, _ = oracle.grid_setup()
    table = rng.uniform(-2e-3, 2e-3, n_params).astype(np.float32)
    mlp = _mlp(rng, 64, n_hidden)
    x = rng.uniform(0.05, 0.95, (4000, 3)).astype(np.float32)
    x = x[_min_preact(oracle, x, table, mlp, 64, n_hidden) > 1e-4][:1500]
    n = len(x)
    assert n == 1500
    gt = rng.uniform(-0.1, 0.1, n).astype(np.float32)
    half, mlp_t, xt = torch.empty(n_params, dtype=torch.float16, device=dev), _t(mlp, dev), _t(x, dev)
    cabi.sdf_table_to_half(_t(table, dev), half)
    probe = cabi.sdf_net(half, mlp_t)
    packed = torch.empty(cabi.sdf_mlp_packed_bytes(probe), dtype=torch.uint8, device=dev)
    cabi.sdf_mlp_pack(probe, packed)
    net = cabi.sdf_net(half, mlp_t, mlp_mode=1, mlp_packed=packed)
    offs = np.array([[0, 0, 0], [1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.float32) * np.float32(delta)
    pts = (x[None] + offs[:, None]).reshape(-1, 3).astype(np.float32)
    r_sdf, r_y1, _ = oracle.sdf_fwd(pts, table, mlp, 64, n_hidden)
    l1, v_s, v_y = oracle.sdf_losses(r_sdf, r_y1, n, 7, gt_sdf=gt, bce_isigma=isg, bce_weight=bce_w, eikonal_weight=0.0, delta=delta)
    tg1, mg1, _ = oracle.sdf_bwd(pts, table, mlp, v_s.reshape(-1).astype(np.float32), v_y.reshape(-1).astype(np.float32), 64, n_hidden)
    g = oracle.sdf_grad_analytic(x, table, mlp, 64, n_hidden).astype(np.float64)
    s7 = r_sdf.reshape(7, n).astype(np.float64)
    gnum = np.stack([s7[1] - s7[2], s7[3] - s7[4], s7[5] - s7[6]], 1) * (0.5 / delta)
    nrm = np.linalg.norm(g, axis=1)
    l2 = eik_w * np.mean((nrm - 1) ** 2) + align_w * np.mean(np.abs(g - gnum))
    c = (eik_w / n) * (2 * (nrm - 1) / nrm)[:, None] * g + (align_w / (3 * n)) * np.sign(g - gnum)
    tg2, mg2 = oracle.sdf_grad_analytic_bwd(x, table, mlp, c.astype(np.float32), 64, n_hidden)
    loss, tg, mg = torch.zeros(1, device=dev), torch.zeros(n_params, device=dev), torch.zeros(len(mlp), device=dev)
    cabi.sdf_train(net, xt, 7, delta, _t(gt, dev), None, isg, bce_w, eik_w, 0.0, loss, tg, mg, None, eikonal_mode=1, align_weight=align_w)
    torch.cuda.synchronize()
    mgc, tgc = mg.cpu().numpy().astype(np.float64), tg.cpu().numpy().astype(np.float64)
    e_l = abs(float(loss) - (l1 + l2)) / abs(l1 + l2)
    e_m, e_t = rel(mgc, mg1 + mg2), rel(tgc, tg1 + tg2)
    e_m2, e_t2 = rel(mgc - mg1, mg2), rel(tgc - tg1, tg2)
    print(f"analytic eikonal vs oracle: loss {e_l:.2e}; total grad mlp {e_m:.2e} table {e_t:.2e}; second-order share mlp {e_m2:.2e} table {e_t2:.2e}")
    assert np.linalg.norm(mg2) > 1e-3 * np.linalg.norm(mg1)
    assert e_l <= 1e-4
    assert e_m <= 1e-3 and e_t <= 1e-3, (e_m, e_t)
    assert e_m2 <= 1e-3 and e_t2 <= 1e-3, (e_m2, e_t2)


def test_gate_compaction_equals_reference_index_select(oracle):
    """gssdf_sdf_gate_compact + gssdf_scatter_rows3 (the step's arrangement of the coupling site) == torch index_select / index_put of the
    gated rows, and the fused kernel on the compact batch == the in-kernel gate on the full batch."""
    from gssdf_b200 import cabi
    dev = _dev()
    rng = np.random.default_rng(4)
    n, live, thr, delta = 5000, 4100, 0.1, 0.01
    x = rng.uniform(0.05, 0.95, (n, 3)).astype(np.float32)
    vis = rng.uniform(0, 0.3, n).astype(np.float32)
    valid = (rng.uniform(0, 1, n) > 0.3).astype(np.uint8)
    w = rng.uniform(0.2, 1.0, n).astype(np.float32)
    sel = np.flatnonzero((vis[:live] > thr) & (valid[:live] != 0))
    n_live = torch.tensor([live], dtype=torch.int32, device=dev)
    idx, xo, wo = torch.full((n,), -7, dtype=torch.int32, device=dev), torch.zeros(n, 3, device=dev), torch.zeros(n, device=dev)
    ng = torch.zeros(1, dtype=torch.int32, device=dev)
    cabi.sdf_gate_compact(n, _t(x, dev), idx, xo, ng, cabi.Workspace(dev), visibilities=_t(vis, dev), visible_thr=thr, valid_mask=_t(valid, dev),
                          weights=_t(w, dev), w_out=wo, n_live=n_live)
    k = int(ng)
    assert k == len(sel) and np.array_equal(idx[:k].cpu().numpy(), sel)
    assert np.array_equal(xo[:k].cpu().numpy(), x[sel]) and np.allclose(wo[:k].cpu().numpy(), w[sel] * vis[sel], rtol=1e-7)
    src = torch.randn(n, 3, device=dev)
    dst = torch.full((n, 3), 5.0, device=dev)
    cabi.scatter_rows3(n, idx, ng, src, dst, n_live=n_live)
    ref = np.full((n, 3), 5.0, np.float32)
    ref[:live] = 0
    ref[sel] = src[:k].cpu().numpy()
    assert np.array_equal(dst.cpu().numpy(), ref)
    # fused kernel: compact batch == in-kernel gate
    n_params, _ = oracle.grid_setup()
    table = rng.uniform(-2e-4, 2e-4, n_params).astype(np.float32)
    mlp = _mlp(rng, 64, 3)
    half, mlp_t = torch.empty(n_params, dtype=torch.float16, device=dev), _t(mlp, dev)
    cabi.sdf_table_to_half(_t(table, dev), half)
    probe = cabi.sdf_net(half, mlp_t)
    packed = torch.empty(cabi.sdf_mlp_packed_bytes(probe), dtype=torch.uint8, device=dev)
    cabi.sdf_mlp_pack(probe, packed)
    net = cabi.sdf_net(half, mlp_t, mlp_mode=1, mlp_packed=packed)
    z = lambda *s: torch.zeros(*s, device=dev)
    la, tga, mga, vxa = z(1), z(n_params), z(len(mlp)), z(n, 3)
    cabi.sdf_train(net, _t(x, dev), 7, delta, None, _t(w, dev), 10.0, 0.0, 0.1, 1e-3, la, tga, mga, vxa, visibilities=_t(vis, dev), visible_thr=thr,
                   n_live=n_live, eikonal_mode=1, align_weight=0.1, valid_mask=_t(valid, dev), n_gate=ng)
    lb, tgb, mgb, vxc, vxb = z(1), z(n_params), z(len(mlp)), z(n, 3), z(n, 3)
    cabi.sdf_train(net, xo, 7, delta, None, wo, 10.0, 0.0, 0.1, 1e-3, lb, tgb, mgb, vxc, n_live=ng, eikonal_mode=1, align_weight=0.1)
    cabi.scatter_rows3(n, idx, ng, vxc, vxb, n_live=n_live)
    torch.cuda.synchronize()
    assert abs(float(la) - float(lb)) <= 1e-5 * abs(float(la)) and float(la) != 0
    assert rel(mgb.cpu().numpy(), mga.cpu().numpy()) <= 1e-4 and rel(tgb.cpu().numpy(), tga.cpu().numpy()) <= 1e-4
    assert rel(vxb.cpu().numpy(), vxa.cpu().numpy()) <= 1e-4


def test_local_map_checkpoint_archive_round_trip(tmp_path):
    """f-4: local_map_checkpoint.pt is libtorch's own module archive (torch::save(local_map_ptr), neural_mapping.cpp:1331-1342): written and
    read back through the shim's module with the reference's parameter names; the fp16 shadow follows the loaded values."""
    import gssdf_shim
    dev = _dev()
    A = gssdf_shim.LocalMapReplay(16, 2, 16, 64, 3, 14.0, 0.1)
    names = A.parameter_names()
    assert names[0] == "encoder_local_map" and "decoder.0.weight" in names and "decoder.8.bias" in names and len(names) == 11
    with torch.no_grad():
        A.encoder_params().uniform_(-0.3, 0.3)
    x = torch.rand(300, 3, device=dev) * 8 - 4
    ya = A.get_sdf(x)[0]
    path = str(tmp_path / "local_map_checkpoint.pt")
    A.save(path)
    B = gssdf_shim.LocalMapReplay(16, 2, 16, 64, 3, 14.0, 0.1)
    assert not torch.equal(B.get_sdf(x)[0], ya)
    B.load(path)
    assert torch.equal(B.encoder_params(), A.encoder_params()) and torch.equal(B.get_sdf(x)[0], ya)
    # the archive is a regular TorchScript-style zip: python can open it too
    m = torch.jit.load(path, map_location="cpu")
    assert dict(m.named_parameters())["encoder_local_map"].shape == A.encoder_params().shape


def test_two_stream_schedule_equals_in_line_schedule():
    """GsSdfStep.overlap only changes WHERE the SDF-only work is enqueued (a second stream beside the render); losses and the flat gradient
    must agree with the in-line schedule up to the order of the float atomics, over several consecutive steps with Adam in between."""
    from gssdf_b200 import octree as OT, parallel, render, scene as S
    dev = _dev()
    rng = np.random.default_rng(5)
    W, H, N, deg = 160, 96, 4000, 3
    sc = S.box_scene(N, deg, seed=0)
    V, K = S.camera(0, W, H)
    cfg = dict(n_levels=16, n_features=2, log2_hashmap_size=19, base_resolution=32, per_level_scale=2.0, hidden_dim=64, n_hidden=3)
    table = (rng.uniform(-1, 1, 16 * 2 * (1 << 19)).astype(np.float32)) * 2e-4
    out = {}
    for overlap in (False, True, "coupling only"):
        torch.manual_seed(11)
        T = render.GsSdfTrainer(N, (deg + 1) ** 2, W, H, dev, 300000, cfg, n_ray_samples=8192, sh_degree=deg, map_size=14.0,
                                normal_weight=0.01, isotropic_weight=0.05)
        T.overlap = bool(overlap)
        T.overlap_ray_stage = overlap is True  # "coupling only": sample generation + [A] stay on the caller's stream
        probe = T.n_mlp
        mlp = torch.from_numpy(np.random.default_rng(6).uniform(-0.2, 0.2, probe).astype(np.float32)).to(dev)
        op_ = np.clip(sc["opacities"], 1e-6, 1 - 1e-6)
        T.load(_t(sc["means"], dev), torch.zeros(N, 3, device=dev), _t(sc["quats"], dev), _t(np.log(sc["scales"]), dev),
               _t(np.log(op_ / (1 - op_)), dev), _t(sc["sh"][:, :1].copy(), dev), _t(sc["sh"][:, 1:].copy(), dev), _t(table[:T.n_table], dev), mlp)
        q = OT.quantize_points(_t(sc["means"], dev) * (2.0 / 14.0), 6)
        tree = OT.OctreeAS.from_quantized_points(q, 6, dev, map_size=14.0)
        T.set_octree(tree)
        n_rays = 500
        r2 = np.random.default_rng(7)
        ro = (r2.uniform(-0.5, 0.5, (n_rays, 3)) * S.BOX).astype(np.float32)
        rend = sc["means"][r2.integers(0, N, n_rays)].astype(np.float32)
        rdep = np.linalg.norm(rend - ro, axis=1).astype(np.float32)
        rdir = ((rend - ro) / rdep[:, None]).astype(np.float32)
        RS = OT.RaySampler(tree, n_rays, dev, 1, 3, 3, 0.1, 0.3, nugget_cap=64 * n_rays, cap=8192)
        gt = torch.rand(1, H, W, 4, device=dev, generator=torch.Generator(dev).manual_seed(3))
        rn = torch.randn(N, 2, device=dev, generator=torch.Generator(dev).manual_seed(4))
        gen = torch.Generator(dev).manual_seed(9)
        rec = []
        DP = parallel.DataParallelStep(T, 1)
        for it in range(4):
            with T.sdf_stage():
                RS.rand_voxel.uniform_(generator=gen); RS.rand_free.uniform_(generator=gen); RS.randn_surface.normal_(generator=gen)
                RS.sample(_t(ro, dev), _t(rdir, dev), _t(rdep, dev), _t(rend, dev))
            if it < 2:  # the step itself: gradients before any optimiser call
                loss, sdf_loss = T.train_step(_t(V[None], dev), _t(K[None], dev), gt, RS.xyz, RS.ray_sdf, rn, ray_n_live=RS.counts)
                torch.cuda.synchronize()
                rec.append((float(loss), float(sdf_loss), T.flat_grad.clone(), int(T.n_gate[0]), int(RS.counts[0])))
                T.adam_all()
            else:       # the way bench.py drives it
                loss, sdf_loss = DP.step(_t(V[None], dev), _t(K[None], dev), gt, RS.xyz, RS.ray_sdf, rn, ray_n_live=RS.counts)
                torch.cuda.synchronize()
                rec.append((float(loss), float(sdf_loss), None, int(T.n_gate[0]), int(RS.counts[0])))
                assert float(T.flat_grad.abs().max()) == 0.0 and T.t_sdf == T.t_splat == it + 1
        torch.cuda.synchronize()
        out[overlap] = (rec, T.params.clone())
    for other in (True, "coupling only"):
        for k, ((l0, s0, g0, n0, c0), (l1, s1, g1, n1, c1)) in enumerate(zip(out[False][0], out[other][0])):
            assert n0 == n1 and c0 == c1 and n0 > 0 and c0 > 0
            # the same step on the same parameters agrees to the order of the float REDs; every Adam step (eps 1e-15: a sign-like update
            # on near-zero gradients) then amplifies that run-to-run noise a little, whatever the schedule
            tol = 1e-4 if k == 0 else 2e-3
            assert abs(l0 - l1) <= 0.1 * tol * abs(l0) and abs(s0 - s1) <= tol * abs(s0), (k, l0, l1, s0, s1)
            if g0 is not None:
                assert rel(g1.cpu().numpy(), g0.cpu().numpy()) < 1e-4
        # parameters after four optimiser steps: equal up to that noise (a sign-like Adam update of a near-zero gradient may flip: a few
        # entries move by ~ lr per step the other way)
        pa, pb = out[False][1].cpu().numpy(), out[other][1].cpu().numpy()
        assert rel(pb, pa) < 1e-3 and float(np.abs(pa - pb).max()) < 0.05, (rel(pb, pa), float(np.abs(pa - pb).max()))


@pytest.mark.parametrize("n,live,p_keep", [(100000, 91000, 0.4), (40000, 40000, 1.0), (40000, 40000, 0.0), (70000, 0, 0.5), (1, 1, 1.0),
                                           (32769, 32769, 0.5), (4096 * 9, 4096 * 9 - 1, 0.5)])
def test_gate_compaction_sizes_and_degenerate_masks(n, live, p_keep):
    """flag -> scan -> gather at sizes on both sides of the single-CTA / chunked scan switch, with all / none / no live rows."""
    from gssdf_b200 import cabi
    dev = _dev()
    rng = np.random.default_rng(n + live)
    x = rng.uniform(0, 1, (n, 3)).astype(np.float32)
    vis = np.where(rng.uniform(0, 1, n) < p_keep, 0.5, 0.01).astype(np.float32)
    sel = np.flatnonzero(vis[:live] > 0.1)
    n_live = torch.tensor([live], dtype=torch.int32, device=dev)
    idx, xo = torch.full((n,), -7, dtype=torch.int32, device=dev), torch.zeros(n, 3, device=dev)
    ng = torch.full((1,), -1, dtype=torch.int32, device=dev)
    cabi.sdf_gate_compact(n, _t(x, dev), idx, xo, ng, cabi.Workspace(dev), visibilities=_t(vis, dev), visible_thr=0.1, n_live=n_live)
    k = int(ng)
    assert k == len(sel)
    assert np.array_equal(idx[:k].cpu().numpy(), sel) and np.array_equal(xo[:k].cpu().numpy(), x[sel])
    src, dst = torch.randn(n, 3, device=dev), torch.full((n, 3), 5.0, device=dev)
    cabi.scatter_rows3(n, idx, ng, src, dst, n_live=n_live)
    ref = np.full((n, 3), 5.0, np.float32)
    ref[:live] = 0
    ref[sel] = src[:k].cpu().numpy()
    assert np.array_equal(dst.cpu().numpy(), ref)


def test_rows_pack_unpack_equal_index_ops():
    """(e) gssdf_rows_pack / gssdf_rows_unpack_add == torch index_select / index_add over the six splat segments, with a device-side row
    count, zero_source, and duplicate rows on the unpack side."""
    from gssdf_b200 import cabi
    dev = _dev()
    g = torch.Generator(dev).manual_seed(3)
    N, widths = 5000, [3, 4, 3, 1, 3, 45]
    offs = [0]
    for w in widths:
        offs.append(offs[-1] + N * w)
    flat = torch.randn(offs[-1] + 7, device=dev, generator=g)
    segments = list(zip(offs[:-1], widths))
    stride = cabi.rows_stride(segments)
    assert stride == 60
    ids = torch.randperm(N, device=dev, generator=g)[:1800].to(torch.int64)
    n_rows = torch.tensor([1500], dtype=torch.int32, device=dev)
    cap_rows = 1700
    packed = torch.full((cap_rows, stride), 7.5, device=dev)
    src = flat.clone()
    cabi.rows_pack(segments, cap_rows, n_rows, ids, flat, packed, zero_source=True)
    torch.cuda.synchronize()
    live = ids[:1500]
    assert torch.equal(packed[:1500, 0].view(torch.int32).to(torch.int64), live)
    col = 1
    for (o, w) in segments:
        seg = src[o:o + N * w].view(N, w)
        assert torch.equal(packed[:1500, col:col + w], seg[live])
        now = flat[o:o + N * w].view(N, w)
        assert float(now[live].abs().max()) == 0.0  # zero_source
        keep = torch.ones(N, dtype=torch.bool, device=dev)
        keep[live] = False
        assert torch.equal(now[keep], seg[keep])
        col += w
    assert float((packed[1500:] - 7.5).abs().max()) == 0.0 and torch.equal(flat[offs[-1]:], src[offs[-1]:])
    # unpack twice (two "ranks" with the same rows) + a duplicate row inside one packed batch
    packed[1499] = packed[0]
    dst = torch.zeros_like(flat)
    cabi.rows_unpack_add(segments, cap_rows, n_rows, dst, packed)
    cabi.rows_unpack_add(segments, cap_rows, n_rows, dst, packed)
    torch.cuda.synchronize()
    col = 1
    for (o, w) in segments:
        want = torch.zeros(N, w, device=dev)
        want.index_add_(0, packed[:1500, 0].view(torch.int32).to(torch.int64), packed[:1500, col:col + w])
        assert torch.allclose(dst[o:o + N * w].view(N, w), 2 * want, rtol=1e-6, atol=1e-6)
        col += w
    # empty batch
    cabi.rows_unpack_add(segments, cap_rows, torch.zeros(1, dtype=torch.int32, device=dev), dst, packed)
