"""Lazy Adam over the SH row groups: the row update (visible rows, replaying the zero-gradient steps each row missed), the catch-up
before the SH forward, the per-window sweep and the replay-only flush must give exactly the bits of the dense update; and a small trainer
run on the lazy path must match the same run with the dense update to within the run-to-run noise of the render."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _visible_sets(rng, N, steps, W):
    """Per step a sorted list of distinct visible rows: rows 0-9 every step, rows 10-19 seen at step 1 and then absent for exactly W
    steps (seen again at W + 2, 2W + 3, ...), an empty set at step 5 and at the sweep step 2W, and a random 15 % of the rest."""
    out = []
    for t in range(1, steps + 1):
        if t in (5, 2 * W):
            out.append(np.zeros(0, np.int64))
            continue
        s = set(range(10))
        if (t - 1) % (W + 1) == 0:
            s |= set(range(10, 20))
        s |= set((20 + rng.choice(N - 20, int(0.15 * (N - 20)), replace=False)).tolist())
        out.append(np.array(sorted(s), np.int64))
    return out


def test_lazy_rows_bit_exact_against_dense():
    from gssdf_b200 import cabi
    dev = _dev()
    W = cabi.ADAM_WINDOW
    rng = np.random.default_rng(0)
    N, K = 3000, 16
    n_geo, n_tail = 4 * N + 3, 5000  # a dense group before the SH segment (odd length: scalar tail) and one after it
    o_dc = n_geo
    o_rest = o_dc + 3 * N
    o_tail = o_rest + 3 * (K - 1) * N
    n = o_tail + n_tail
    lr_geo, lr_dc, lr_rest, lr_tail = 1e-3, 2.5e-3, 2.5e-3 / 20, 5e-3
    dense_groups = [(0, n_geo, lr_geo, False), (o_dc, 3 * N, lr_dc, False), (o_rest, 3 * (K - 1) * N, lr_rest, False), (o_tail, n_tail, lr_tail, False)]
    lazy_groups = [(0, n_geo, lr_geo, False, 0), (o_dc, 3 * N, lr_dc, False, 3), (o_rest, 3 * (K - 1) * N, lr_rest, False, 3 * (K - 1)),
                   (o_tail, n_tail, lr_tail, False, 0)]
    g0 = torch.Generator(dev).manual_seed(1)
    P = torch.randn(n, device=dev, generator=g0)
    M = torch.randn(n, device=dev, generator=g0) * 1e-3
    V = torch.rand(n, device=dev, generator=g0) * 1e-6
    D = dict(p=P.clone(), m=M.clone(), v=V.clone(), g=torch.zeros(n, device=dev))
    L = dict(p=P.clone(), m=M.clone(), v=V.clone(), g=torch.zeros(n, device=dev))
    last = torch.zeros(N, dtype=torch.int32, device=dev)
    replay = cabi.AdamReplay(last)
    counts = torch.zeros(cabi.COUNTS_INTS, dtype=torch.int32, device=dev)
    cam_ids = torch.zeros(N, dtype=torch.int64, device=dev)  # stands in for an empty row list

    def sh_views(b):
        return b[o_dc:o_rest].view(N, 1, 3), b[o_rest:o_tail].view(N, K - 1, 3)

    def rows(b, ids):
        dc, rest = sh_views(b)
        return torch.cat([dc[ids].reshape(len(ids), -1), rest[ids].reshape(len(ids), -1)], 1)

    steps = 2 * W + 10
    vis = _visible_sets(rng, N, steps, W)
    specials = [0.0, -0.0, 1e-40, -1e-40, 1.4e-45, 3e-39]  # +-0 and subnormal gradients
    checked_rows = 0
    for t in range(1, steps + 1):
        ids_np = vis[t - 1]
        ids = torch.from_numpy(ids_np).to(dev)
        counts[0] = len(ids_np)
        # (b) catch-up before the SH forward of step t: the rows it reads hold their step t-1 values
        if t > 1:
            cabi.adam_step(L["p"], L["g"], L["m"], L["v"], lazy_groups[1:3], t - 1, replay=replay, row_ids=ids if len(ids_np) else cam_ids,
                           row_count=counts, row_cap=N, replay_only=True)
        if len(ids_np):
            for k in ("p", "m", "v"):
                assert torch.equal(rows(L[k], ids), rows(D[k], ids)), (t, k)
            assert bool((last[ids] == t - 1).all())
            checked_rows += len(ids_np)
        # step t's gradient: dense groups everywhere, SH rows only where visible (the rest hold +0, as after zero_grad)
        g = torch.zeros(n, device=dev)
        g[:n_geo] = torch.randn(n_geo, device=dev, generator=g0)
        g[o_tail:] = torch.randn(n_tail, device=dev, generator=g0)
        if len(ids_np):
            r = torch.randn(len(ids_np), 3 * K, device=dev, generator=g0) * 1e-2
            r[: min(3, len(ids_np))] = 0.0  # visible rows with all-zero gradients
            flat = r.view(-1)
            pick = torch.from_numpy(rng.choice(flat.numel(), min(64, flat.numel()), replace=False)).to(dev)
            flat[pick] = torch.tensor(specials, device=dev).repeat(11)[: pick.numel()]
            dc_g, rest_g = sh_views(g)
            dc_g[ids] = r[:, :3].reshape(-1, 1, 3)
            rest_g[ids] = r[:, 3:].reshape(-1, K - 1, 3)
        D["g"].copy_(g)
        L["g"].copy_(g)
        gs = 0.5 if t % 3 == 0 else 1.0
        replay.push(t, lr_dc, lr_rest)
        cabi.adam_step(D["p"], D["g"], D["m"], D["v"], dense_groups, t, grad_scale=gs)
        sweep = t % W == 0
        cabi.adam_step(L["p"], L["g"], L["m"], L["v"], lazy_groups, t, grad_scale=gs, replay=replay,
                       row_ids=None if sweep else (ids if len(ids_np) else cam_ids), row_count=counts, row_cap=N)
        if sweep:
            for k in ("p", "m", "v", "g"):
                assert torch.equal(L[k], D[k]), (t, k)
            assert bool((last == t).all())
        else:
            assert torch.equal(L["p"][:n_geo], D["p"][:n_geo]) and torch.equal(L["p"][o_tail:], D["p"][o_tail:])
            if len(ids_np):
                assert bool((last[ids] == t).all())
    assert checked_rows > 0
    # (c) flush: every row brought to the last step; then everything, the zeroed gradients included, is identical
    cabi.adam_step(L["p"], L["g"], L["m"], L["v"], lazy_groups[1:3], steps, replay=replay, replay_only=True)
    torch.cuda.synchronize()
    for k in ("p", "m", "v", "g"):
        assert torch.equal(L[k], D[k]), k
    assert float(L["g"].abs().max()) == 0.0
    assert bool((last == steps).all())


def _trainer_run(dev, n_steps, dense):
    """A small GsSdfTrainer run cycling 8 cameras; dense=True drives the optimiser through cabi.adam_step with every group dense."""
    from gssdf_b200 import cabi, render
    from gssdf_b200 import octree as OT
    from gssdf_b200 import scene as S
    W_, H_, N, deg = 160, 96, 4000, 3
    sc = S.box_scene(N, deg, seed=0)
    cfg = dict(n_levels=16, n_features=2, log2_hashmap_size=19, base_resolution=32, per_level_scale=2.0, hidden_dim=64, n_hidden=3)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    T = render.GsSdfTrainer(N, (deg + 1) ** 2, W_, H_, dev, 300000, cfg, n_ray_samples=8192, sh_degree=deg, map_size=14.0,
                            normal_weight=0.01, isotropic_weight=0.05)
    table = (np.random.default_rng(5).uniform(-1, 1, T.n_table).astype(np.float32)) * 2e-4
    mlp = t(np.random.default_rng(6).uniform(-0.2, 0.2, T.n_mlp).astype(np.float32))
    op_ = np.clip(sc["opacities"], 1e-6, 1 - 1e-6)
    T.load(t(sc["means"]), torch.zeros(N, 3, device=dev), t(sc["quats"]), t(np.log(sc["scales"])), t(np.log(op_ / (1 - op_))),
           t(sc["sh"][:, :1].copy()), t(sc["sh"][:, 1:].copy()), t(table), mlp)
    tree = OT.OctreeAS.from_quantized_points(OT.quantize_points(t(sc["means"]) * (2.0 / 14.0), 6), 6, dev, map_size=14.0)
    T.set_octree(tree)
    r2 = np.random.default_rng(7)
    n_rays = 500
    ro = (r2.uniform(-0.5, 0.5, (n_rays, 3)) * S.BOX).astype(np.float32)
    rend = sc["means"][r2.integers(0, N, n_rays)].astype(np.float32)
    rdep = np.linalg.norm(rend - ro, axis=1).astype(np.float32)
    rdir = ((rend - ro) / rdep[:, None]).astype(np.float32)
    RS = OT.RaySampler(tree, n_rays, dev, 1, 3, 3, 0.1, 0.3, nugget_cap=64 * n_rays, cap=8192)
    cams = [S.camera(i, W_, H_) for i in range(8)]
    gt = torch.rand(1, H_, W_, 4, device=dev, generator=torch.Generator(dev).manual_seed(3))
    rn = torch.randn(N, 2, device=dev, generator=torch.Generator(dev).manual_seed(4))
    gen = torch.Generator(dev).manual_seed(9)
    if dense:
        T.scene["raw"]["sh_catch_up"] = None  # every row is current after every dense step
    for it in range(n_steps):
        RS.rand_voxel.uniform_(generator=gen); RS.rand_free.uniform_(generator=gen); RS.randn_surface.normal_(generator=gen)
        RS.sample(t(ro), t(rdir), t(rdep), t(rend))
        V, K = cams[it % 8]
        T.train_step(t(V[None]), t(K[None]), gt, RS.xyz, RS.ray_sdf, rn, ray_n_live=RS.counts)
        if dense:
            T.t_sdf += 1
            T.t_splat += 1
            cabi.adam_step(T._params, T.flat_grad, T._exp_avg, T._exp_avg_sq, [g[:4] for g in T.splat_groups] + T.sdf_groups, T.t_sdf,
                           table_half=T.table_half, net=T._net, mlp_packed=T.mlp_packed)
        else:
            T.adam_all()
    out = T.params.clone()
    torch.cuda.synchronize()
    assert float(T.flat_grad.abs().max()) == 0.0
    if not dense:
        assert bool((T.sh_last == n_steps).all())
    return out.cpu().numpy()


def test_trainer_lazy_sh_matches_dense_update():
    """Through one sweep (ADAM_WINDOW steps) and past it. The raster's float REDs are order-nondeterministic and every Adam step (eps
    1e-15) amplifies that noise, so two dense runs differ too: the lazy run must stay within twice the measured dense-vs-dense
    difference."""
    from gssdf_b200 import cabi
    dev = _dev()
    n_steps = cabi.ADAM_WINDOW + 6
    a = _trainer_run(dev, n_steps, dense=True)
    b = _trainer_run(dev, n_steps, dense=True)
    c = _trainer_run(dev, n_steps, dense=False)
    rel = lambda x, y: float(np.linalg.norm(x - y) / max(np.linalg.norm(y), 1e-30))
    noise, noise_max = rel(b, a), float(np.abs(b - a).max())
    assert rel(c, a) <= 2 * noise + 1e-6 and float(np.abs(c - a).max()) <= 2 * noise_max + 1e-6, (rel(c, a), noise, float(np.abs(c - a).max()), noise_max)
