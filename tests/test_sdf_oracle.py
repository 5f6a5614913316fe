"""CPU checks of the SDF oracle (oracle/sdf_oracle.c): fp16 emulation against numpy's IEEE binary16, grid
geometry against the numbers SURVEY.md section 8a quotes from tiny-cuda-nn (15 269 888 parameters), the restated
backward against finite differences. tiny-cuda-nn ships no tests, so this is the only pin (parity UNPINNED
against reference outputs, see the file header)."""
import numpy as np
import pytest


def _net(rng, hidden=64, n_hidden=3, in_dim=32):
    dims = [in_dim] + [hidden] * (1 + n_hidden) + [2]
    ps = []
    for k, o in zip(dims[:-1], dims[1:]):
        b = 1 / np.sqrt(k)
        ps += [rng.uniform(-b, b, o * k), rng.uniform(-b, b, o)]
    return np.concatenate(ps).astype(np.float32), dims


def test_half_emulation_matches_ieee(oracle):
    rng = np.random.default_rng(0)
    x = (rng.standard_normal(200000) * 10.0 ** rng.integers(-9, 6, 200000)).astype(np.float32)
    x = np.concatenate([x, np.array([0, -0.0, 65504, 65519.9, 65520, 1e-8, 2.98e-8, 2.99e-8, 6e-8, 6.1e-5, np.inf, -np.inf], np.float32)])
    with np.errstate(over="ignore"):
        assert np.array_equal(oracle.f32_to_f16_bits(x), x.astype(np.float16).view(np.uint16))


def test_grid_geometry(oracle):
    n, off = oracle.grid_setup()  # config/base.yaml:8-10 + encoding_map.cpp:15-23
    assert n == 15269888 and list(off[:4]) == [0, 32768, 32768 + 262144, 32768 + 262144 + 524288] and off[-1] == 7634944


def test_hashgrid_forward_is_trilinear_and_fp16(oracle):
    rng = np.random.default_rng(1)
    n_params, _ = oracle.grid_setup()
    table = rng.uniform(-0.5, 0.5, n_params).astype(np.float32)
    x = rng.uniform(0.05, 0.95, (300, 3)).astype(np.float32)
    feat, dy = oracle.hashgrid_fwd(x, table, want_dy_dx=True)
    assert np.array_equal(feat, feat.astype(np.float16).astype(np.float32))  # outputs are fp16-exact
    assert np.abs(feat).max() <= 0.5 + 1e-3 and np.abs(feat).mean() > 0.05
    # level 0 is a dense 32^3 grid (scale 31): compare with an independent numpy trilinear interpolation
    t0 = table[: 32768 * 2].astype(np.float16).astype(np.float64).reshape(32, 32, 32, 2)  # [z][y][x][f]
    pos = x.astype(np.float64) * 31 + 0.5
    i0 = np.floor(pos).astype(int)
    fr = pos - i0
    ref = np.zeros((len(x), 2))
    for c in range(8):
        o = [(c >> d) & 1 for d in range(3)]
        w = np.prod([fr[:, d] if o[d] else 1 - fr[:, d] for d in range(3)], 0)
        ref += w[:, None] * t0[(i0[:, 2] + o[2]) % 32, (i0[:, 1] + o[1]) % 32, (i0[:, 0] + o[0]) % 32]
    np.testing.assert_allclose(feat[:, :2], ref, atol=2e-3)  # fp16 accumulation of 8 terms
    # dy_dx vs finite differences of the (fp16-rounded) forward at the coarse levels
    eps = 2e-3
    for d in range(3):
        xp, xm = x.copy(), x.copy()
        xp[:, d] += eps
        xm[:, d] -= eps
        fd = (oracle.hashgrid_fwd(xp, table) - oracle.hashgrid_fwd(xm, table)) / (xp[:, d] - xm[:, d])[:, None]
        same_cell = np.floor(xp * 31 + 0.5)[:, d] == np.floor(xm * 31 + 0.5)[:, d]
        np.testing.assert_allclose(dy[same_cell][:, :2, d], fd[same_cell][:, :2], atol=0.3, rtol=5e-2)


@pytest.mark.parametrize("hidden,n_hidden", [(64, 3), (32, 1)])
def test_mlp_backward_is_derivative(oracle, hidden, n_hidden):
    rng = np.random.default_rng(2)
    params, dims = _net(rng, hidden, n_hidden)
    x = rng.standard_normal((40, 32)).astype(np.float32)
    v = rng.standard_normal((40, 2))
    d_in, d_p = oracle.mlp_bwd(x, dims, params, v)
    loss = lambda xx, pp: float((oracle.mlp_fwd(xx, dims, pp) * v).sum())
    for trial in range(3):
        # a random direction over all 14 k parameters has norm ~120, so the step must be tiny for the ReLU network to
        # stay in one linear region; use the realised fp32 step in the analytic side
        eps = 1e-6
        dp = rng.standard_normal(params.shape)
        pp, pm = (params + eps * dp).astype(np.float32), (params - eps * dp).astype(np.float32)
        fd = (loss(x, pp) - loss(x, pm)) / (2 * eps)
        an = float((d_p * ((pp.astype(np.float64) - pm.astype(np.float64)) / (2 * eps))).sum())
        assert abs(fd - an) <= 2e-3 * max(abs(fd), 1), (fd, an)
        dx = rng.standard_normal(x.shape)
        eps = 1e-5
        xp, xm = (x + eps * dx).astype(np.float32), (x - eps * dx).astype(np.float32)
        fd = (loss(xp, params) - loss(xm, params)) / (2 * eps)
        an = float((d_in * ((xp.astype(np.float64) - xm.astype(np.float64)) / (2 * eps))).sum())
        assert abs(fd - an) <= 2e-3 * max(abs(fd), 1), (fd, an)


def test_sdf_chain_table_gradient(oracle):
    """table gradient of the chained oracle: sum over the table equals the sum of weights x cotangent (partition of unity),
    and only touched entries are non-zero."""
    rng = np.random.default_rng(3)
    n_params, off = oracle.grid_setup()
    table = rng.uniform(-0.5, 0.5, n_params).astype(np.float32)
    params, dims = _net(rng)
    x = rng.uniform(0.05, 0.95, (200, 3)).astype(np.float32)
    tg, d_mlp, dx = oracle.sdf_bwd(x, table, params, np.ones(200), np.zeros(200))
    feat = oracle.hashgrid_fwd(x, table)
    d_feat, _ = oracle.mlp_bwd(feat, dims, params, np.stack([np.ones(200), np.zeros(200)], 1))
    per_level = tg.reshape(-1, 2)
    for lvl in (0, 1, 5, 15):
        seg = per_level[off[lvl]:off[lvl + 1]].sum(0)
        np.testing.assert_allclose(seg, d_feat[:, 2 * lvl:2 * lvl + 2].sum(0), rtol=3e-3, atol=3e-4)  # fp16 rounding of w and g
    assert (tg != 0).sum() <= 200 * 16 * 8 * 2 and np.isfinite(dx).all() and np.abs(dx).max() > 0


def test_analytic_gradient_double_backward_matches_torch_autograd(oracle):
    """The closed-form chains of oracle.sdf_grad_analytic(_bwd) (first backward seeded with w_out[0]; r = dy_dx . c; forward-like
    q-chain; outer products; kernel_grid_backward_input_backward_grid) against torch.autograd double backward of an independent
    fp64 torch restatement (trilinear grid lookup + Linear/ReLU stack). fp16 rounding points switched off for this check."""
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(0)
    n_params, _ = oracle.grid_setup()
    table = rng.uniform(-1e-2, 1e-2, n_params).astype(np.float32)
    dims, ps = [32, 64, 64, 64, 64, 2], []
    for k, o in zip(dims[:-1], dims[1:]):
        b = 1 / np.sqrt(k)
        ps += [rng.uniform(-b, b, o * k), rng.uniform(-b, b, o)]
    mlp = np.concatenate(ps).astype(np.float32)
    n = 64
    x = rng.uniform(0.05, 0.95, (n, 3)).astype(np.float32)
    c = rng.standard_normal((n, 3)).astype(np.float32)
    oracle.set_half_rounding(False)
    try:
        g = oracle.sdf_grad_analytic(x, table, mlp)
        tg, mg = oracle.sdf_grad_analytic_bwd(x, table, mlp, c)
    finally:
        oracle.set_half_rounding(True)
    # torch restatement
    idx = torch.from_numpy(oracle.grid_corner_indices(x))  # [n,16,8]
    xt = torch.tensor(x, dtype=torch.float64, requires_grad=True)
    tab = torch.tensor(table, dtype=torch.float64, requires_grad=True)
    par = torch.tensor(mlp, dtype=torch.float64, requires_grad=True)
    feats = []
    for lvl in range(16):
        scale = float(np.float32(np.exp2(np.float32(lvl)) * 32 - 1))
        # the kernels compute pos = fmaf(scale, x, 0.5) in fp32 (one rounding): at the fine levels the fractional part keeps only
        # a few bits, so the torch restatement must start from the same fp32 value (derivative: scale)
        pos32 = (np.float64(np.float32(scale)) * x.astype(np.float64) + 0.5).astype(np.float32)
        fr0 = torch.tensor((pos32 - np.floor(pos32)).astype(np.float64))
        fr = fr0 + (xt - xt.detach()) * scale
        f = 0
        for corner in range(8):
            w = 1
            for d in range(3):
                w = w * (fr[:, d] if (corner >> d) & 1 else 1 - fr[:, d])
            e = idx[:, lvl, corner]
            f = f + w[:, None] * torch.stack([tab[e], tab[e + 1]], 1)
        feats.append(f)
    a, o = torch.cat(feats, 1), 0
    for li, (k, q) in enumerate(zip(dims[:-1], dims[1:])):
        W, b = par[o:o + q * k].view(q, k), par[o + q * k:o + q * k + q]
        o += q * k + q
        a = a @ W.T + b
        if li < len(dims) - 2:
            a = torch.relu(a)
    sdf = a[:, 0]
    (gt,) = torch.autograd.grad(sdf.sum(), xt, create_graph=True)
    assert np.allclose(gt.detach().numpy(), g, rtol=2e-4, atol=2e-4 * np.abs(g).max())
    (gt * torch.tensor(c, dtype=torch.float64)).sum().backward()
    r_mg, r_tg = par.grad.numpy(), tab.grad.numpy()
    assert np.linalg.norm(mg - r_mg) <= 1e-4 * np.linalg.norm(r_mg), np.linalg.norm(mg - r_mg) / np.linalg.norm(r_mg)
    assert np.linalg.norm(tg - r_tg) <= 1e-4 * np.linalg.norm(r_tg), np.linalg.norm(tg - r_tg) / np.linalg.norm(r_tg)


def _tcnn_golden():
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tcnn_grid_ref.npz"))
    rng = np.random.default_rng(int(g["seed"]))
    table = rng.uniform(-0.5, 0.5, int(g["n_params"])).astype(np.float32)  # first draw of gen_golden_tcnn.py
    return g, table, dict(L=int(g["cfg"][0]), F=2, log2_hashmap=int(g["cfg"][1]), base_res=int(g["cfg"][2]), per_level_scale=2.0)


def test_oracle_grid_matches_tiny_cuda_nn_kernels(oracle):
    """The hash-grid restatement against outputs of tiny-cuda-nn's OWN kernels (kernel_grid, kernel_grid_backward,
    kernel_grid_backward_input, kernel_grid_backward_input_backward_grid/_dLdoutput from the reference's grid.h, instantiated by
    oracle/ref_tcnn_grid_driver.cu and run on an H100: tests/golden/tcnn_grid_ref.npz, generator oracle/gen_golden_tcnn.py)."""
    g, table, cfg = _tcnn_golden()
    x, n_params = g["x"], int(g["n_params"])
    assert oracle.grid_setup(**{k: cfg[k] for k in ("L", "F", "log2_hashmap", "base_res", "per_level_scale")})[0] == n_params
    feat, dy = oracle.hashgrid_fwd(x, table, want_dy_dx=True, **cfg)
    assert np.array_equal(feat, g["enc"]), "encoded features must be bit-identical (fp16 values)"
    assert np.allclose(dy, g["dy_dx"], rtol=1e-6, atol=1e-6 * np.abs(g["dy_dx"]).max())
    # first backward: table gradient (the reference accumulates with half atomics: rounding at every add) and dL/dx
    tg, dx = oracle.hashgrid_bwd(x, g["dL_dy"], n_params, dy, **cfg)
    ref_tg = np.zeros(n_params)
    ref_tg[g["grid_grad_idx"]] = g["grid_grad_val"].astype(np.float64) / 128.0
    assert np.linalg.norm(tg - ref_tg) <= 2e-3 * np.linalg.norm(ref_tg)
    assert set(np.nonzero(tg)[0]) >= set(g["grid_grad_idx"].tolist())  # same touched entries (up to exact zeros)
    assert np.allclose(dx, g["dL_dx_scaled"] / 128.0, rtol=2e-5, atol=1e-6 * np.abs(g["dL_dx_scaled"]).max() / 128.0)
    # double backward
    tg2, r = oracle.hashgrid_bwd_bwd(x, g["cc"], g["dL_dy"], n_params, dy, **cfg)
    ref_tg2 = np.zeros(n_params)
    ref_tg2[g["grid_grad2_idx"]] = g["grid_grad2_val"].astype(np.float64) / 128.0
    # cc ~ N(0,1) times the level scale (up to 1e6) overflows the (half) weight at the finest levels in BOTH (inf / nan entries); the
    # reference additionally saturates when its half-precision running sum passes 65504, which an fp64 accumulator does not
    fin = np.isfinite(ref_tg2) & np.isfinite(tg2)
    touched = (ref_tg2 != 0) | (tg2 != 0)
    assert (np.isfinite(ref_tg2) != np.isfinite(tg2))[touched].mean() <= 0.02
    assert fin[touched].mean() > 0.5
    small = fin & (np.abs(ref_tg2) < 100.0)  # entries far from the half range limit (65504 / 128)
    assert np.linalg.norm(tg2[small] - ref_tg2[small]) <= 2e-3 * np.linalg.norm(ref_tg2[small])
    ulp_off = np.abs(r - g["dL_ddLdy"]) > 0
    assert ulp_off.mean() <= 2e-3 and np.allclose(r, g["dL_ddLdy"], rtol=2e-3, atol=0)  # fp32 sum order: a half ulp on isolated entries
