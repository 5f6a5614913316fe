"""The normal-consistency term on the median depth (GsTrainer(depth_type=), DESIGN 7o) on the GPU: the loss kernel on a stride-1
render_median buffer at 1080p against fp64, the raster backward with a nonzero v_render_median against the fp64 block oracle, a joint
step's median cotangent against fp64 autograd of the reference expression on the step's own render, depth_type 0 launching what the
default launches, no added host synchronisation, and the box room end to end."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from raster_block_oracle import backward, forward, split_record  # noqa: E402
from raster_blocks import all_scenes  # noqa: E402
from test_gpu_deep_tiles import _dev, _Raster, _t  # noqa: E402
from test_gpu_gs_train import room  # noqa: E402,F401 (the box-room fixture)
from test_gpu_raster_blocks import MARGIN, _counts, _label, _ratio  # noqa: E402
from test_gpu_round2 import _depth_to_normal_ref  # noqa: E402
from test_raster_blocks_host import BWD_NAMES, oracle_refs  # noqa: E402


def test_loss_kernel_on_the_median_buffer_at_1080p():
    """neural_mapping.cpp:243-266 with render_median [1,H,W,1] (stride 1) as the depth and v_render_median as the cotangent, at
    1920x1080: loss within 1e-5 relative, dL/d median within 1e-4 of its largest entry of the fp64 restatement."""
    from gssdf_b200 import cabi
    from gssdf_b200 import scene as S
    dev = _dev()
    W, H = 1920, 1080
    g = torch.Generator("cpu").manual_seed(W * H)
    Vn, Kn = S.camera(5, W, H)
    depth32 = (1.0 + torch.rand(H, W, 1, generator=g, dtype=torch.float64) * 2).float()
    depth32[200:230, 400:470] = 0.0  # empty pixels: degenerate stencils
    alpha32 = torch.rand(H, W, 1, generator=g, dtype=torch.float64).float()
    rn32 = torch.nn.functional.normalize(torch.randn(H, W, 3, generator=g, dtype=torch.float64), dim=-1).float()
    w = 0.01
    V, K = torch.from_numpy(Vn).double(), torch.from_numpy(Kn).double()
    depth = depth32.double().requires_grad_(True)
    alpha = alpha32.double()
    dn = _depth_to_normal_ref(depth, V, K) * alpha
    ref = w * (alpha.square().squeeze(-1) - (dn * rn32.double()).sum(-1).nan_to_num()).mean()
    ref.backward()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    med = depth32.to(dev).view(1, H, W, 1).contiguous()
    v_med = torch.zeros(1, H, W, 1, device=dev)
    loss = torch.zeros(1, device=dev)
    cabi.normal_consistency_loss(1, W, H, t(Vn[None]), t(Kn[None]), med, 1, alpha32.to(dev).view(1, H, W, 1), rn32.to(dev).view(1, H, W, 3),
                                 w, loss, v_depth=v_med, v_depth_stride=1, v_out_normals=torch.zeros(1, H, W, 3, device=dev))
    torch.cuda.synchronize()
    assert abs(float(loss) - float(ref)) <= 1e-5 * abs(float(ref))
    gd, gr = v_med[0, ..., 0].cpu().double(), depth.grad[..., 0]
    err = float((gd - gr).abs().max())
    print(f"median normal term 1080p: loss {float(loss):.9e} vs {float(ref):.9e}; dL/d median error {err:.3e} of {float(gr.abs().max()):.3e}")
    assert err <= 1e-4 * float(gr.abs().max())


# ---- the raster backward with a median cotangent -------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def median_blocks(oracle):
    """The block scenes of test_gpu_raster_blocks with a nonzero v_render_median on the pixels whose T-vs-0.5 margin clears MARGIN (the
    only pixels where the median splat is not a rounding decision), and the fp64 backward of those cotangents from the f32 oracle state."""
    out = []
    for sc in all_scenes():
        ref = oracle_refs(oracle, sc)
        f = forward(sc, ref["off"], ref["flat"])
        ct = dict(ref["ct"])
        rng = np.random.default_rng(sc["W"] * 131 + sc["H"] + sc["C"])
        clear = np.asarray(f["median_margin"]).reshape(sc["C"], sc["H"], sc["W"]) > MARGIN
        scale = float(np.abs(ct["v_render_depths"]).max()) or 1.0
        vm = rng.uniform(-1.0, 1.0, clear.shape) * scale * clear
        ct["v_render_median"] = np.ascontiguousarray(vm[..., None], np.float32)
        b = backward(sc, ref["off"], ref["flat"], ref["r32"], ct, f["N"])
        out.append(dict(sc=sc, ref=ref, ct=ct, clear=clear, rec=split_record(b["rec"], sc["ray_transforms"]),
                        A=split_record(b["A"], np.abs(sc["ray_transforms"]))))
    return out


def test_raster_backward_with_a_median_cotangent(median_blocks):
    """Every gradient entry within C_ULP * 2^-24 * A (test_gpu_raster_blocks' bar) of the fp64 backward, and the median cotangent moves
    the gradients (against the run with it zeroed)."""
    dev = _dev()
    worst, n_clear, moved = 0.0, 0, 0.0
    for B in median_blocks:
        sc, ref = B["sc"], B["ref"]
        n_clear += int(B["clear"].sum())
        assert (np.asarray(B["ct"]["v_render_median"])[..., 0][~B["clear"]] == 0).all()
        n = len(ref["flat"])
        off, flat = _t(ref["off"], dev), _t(ref["flat"], dev)
        R = _Raster(dev, sc, n)
        g = R.bwd(_counts(dev, sc, n), off, flat, ref["r32"], B["ct"], reuse_fwd=False)
        for k in BWD_NAMES:
            worst = max(worst, _ratio(g[k], B["rec"][k], B["A"][k], f"{_label(sc)} median {k}"))
        g0 = R.bwd(_counts(dev, sc, n), off, flat, ref["r32"], dict(B["ct"], v_render_median=np.zeros_like(B["ct"]["v_render_median"])),
                   reuse_fwd=False)
        moved = max(moved, max(float(np.abs(np.asarray(g[k], np.float64) - np.asarray(g0[k], np.float64)).max()) for k in BWD_NAMES))
    print(f"median cotangent on {n_clear} pixels: worst |err| / (2^-24 A) = {worst:.3g}; largest gradient change {moved:.3e}")
    assert n_clear > 0 and moved > 0.0


# ---- the joint step ----------------------------------------------------------------------------------------------------------------
def _trainer(room, depth_type, iters=12, seed=2, **kw):
    import test_gpu_gs_train as GS
    S_ = GS._sdf_trainer(room, 100, seed=seed)
    c2w = GS._poses(6, 5)
    return GS._gs_trainer(room, S_, (c2w, GS._images(c2w)), iters, refine_gs_struct_start_iter=3, depth_type=depth_type, **kw)


def test_joint_step_median_cotangent_matches_fp64(room):
    """After the normal term switches on (iteration 4): v_render_median of the step equals fp64 autograd of the reference expression on
    the step's own render_median, alphas and normals; nothing reaches the expected-depth channel of the colour cotangent (the depth
    weight is 0); and a backward without the term leaves v_render_median zero."""
    G = _trainer(room, 1)
    G.run_color_init()
    G.start_rates()
    for i in range(5):
        G.step(i)
    T = G.T
    R = T.R
    torch.cuda.synchronize()
    H, W = R.H, R.W
    V, K = G.viewmats.double().cpu(), G.Ks[0].double().cpu()
    vm = R.v_r["median"][0].double().cpu()
    # the camera of iteration 4
    cam = G.perm[4 % G.train_num]
    med = R.r["render_median"][0].double().cpu().requires_grad_(True)
    alpha = R.r["render_alphas"][0].double().cpu()
    rn = R.out_normals[0].double().cpu()
    dn = _depth_to_normal_ref(med, V[cam], K) * alpha
    ref = G.normal_w * (alpha.square().squeeze(-1) - (dn * rn).sum(-1).nan_to_num()).mean()
    ref.backward()
    err = float((vm - med.grad).abs().max())
    print(f"joint step: dL/d median error {err:.3e} of {float(med.grad.abs().max()):.3e}")
    assert float(med.grad.abs().max()) > 0
    assert err <= 1e-4 * float(med.grad.abs().max())
    assert float(R.v_out_colors[..., 3].abs().max()) == 0.0
    # a backward without the term clears the median cotangent
    sc = T.scene
    R.backward(sc["means"], sc["quats"], sc["scales"], sc["opacities"], sc["sh"], G.viewmats[cam:cam + 1], G.Ks, G.gt, zero_grads=False,
               raw=sc["raw"], w_rgb=T.rgb_w, w_depth=0.0, w_dssim=T.dssim_w, projection_bwd=False, median_depth=True)
    torch.cuda.synchronize()
    assert float(R.v_r["median"].abs().max()) == 0.0


def _record_calls(monkeypatch):
    """Every cabi call of the step as (name, its scalar arguments)"""
    from gssdf_b200 import cabi
    calls = []
    for name in dir(cabi):
        fn = getattr(cabi, name)
        if name.startswith("_") or not callable(fn) or isinstance(fn, type) or getattr(fn, "__module__", None) != cabi.__name__:
            continue

        def wrap(*a, _fn=fn, _name=name, **kw):
            calls.append((_name, tuple(v for v in list(a) + sorted(kw.items()) if isinstance(v, (bool, int, float, str)))))
            return _fn(*a, **kw)
        monkeypatch.setattr(cabi, name, wrap)
    return calls


def test_depth_type_0_launches_what_the_default_launches(room, monkeypatch):
    """Joint iterations 4-7 of 8 (the normal term on, no densification callback) make the same library calls with the same normal-term
    arguments with depth_type=0 as without the argument; depth_type=1 makes the same calls with the median as the depth."""
    seqs = {}
    for label, kw in (("default", {}), ("0", dict(depth_type=0)), ("1", dict(depth_type=1))):
        import test_gpu_gs_train as GS
        S_ = GS._sdf_trainer(room, 100, seed=2)
        c2w = GS._poses(6, 5)
        G = GS._gs_trainer(room, S_, (c2w, GS._images(c2w)), 8, refine_gs_struct_start_iter=3, **kw)
        G.run_color_init()
        G.start_rates()
        for i in range(4):
            G.step(i)
        with monkeypatch.context() as m:  # the second half (no densification callback), the normal term on
            calls = _record_calls(m)
            for i in range(4, 8):
                G.step(i)
        torch.cuda.synchronize()
        seqs[label] = calls
    # the splat count (and so every capacity argument) differs between two SDF stages: the call sequences are compared by name, and the
    # normal term's calls by their scalar arguments without raw device pointers (out_colors + 12)
    names = lambda seq: [n for n, _ in seq]
    nc = lambda seq: [tuple(x for x in a if not (isinstance(x, int) and not isinstance(x, bool) and x > 1 << 40))
                      for n, a in seq if n == "normal_consistency_loss"]
    assert names(seqs["default"]) == names(seqs["0"]) == names(seqs["1"])
    assert nc(seqs["default"]) == nc(seqs["0"]) and len(nc(seqs["0"])) == 4
    assert all(4 in a for a in nc(seqs["0"])) and all(4 not in a for a in nc(seqs["1"]))  # the depth stride: 4 (out_colors), 1 (median)


def test_median_term_adds_no_host_synchronisation(room):
    """Iterations with the median-depth normal term on run under torch.cuda.set_sync_debug_mode("error"), with the densifier's reads
    allowed as in test_gpu_gs_train."""
    G = _trainer(room, 1, iters=16)
    D = G.D

    def allowed(fn, due=lambda *a: True):  # the reads test_iterations_synchronise_only_where_the_reference_reads_back allows
        def wrapped(*a, **kw):
            if not due(*a):
                return fn(*a, **kw)
            torch.cuda.set_sync_debug_mode("default")
            try:
                return fn(*a, **kw)
            finally:
                torch.cuda.set_sync_debug_mode("error")
        return wrapped
    D.prune_nan_gs = allowed(D.prune_nan_gs)
    D.prune_invisible_gs = allowed(D.prune_invisible_gs, lambda it: it > 0 and it % D.num_train_data == 0)
    D.grow_gs, D.prune_gs = allowed(D.grow_gs), allowed(D.prune_gs)
    G.run_color_init()
    G.start_rates()
    G.step(0)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for i in range(1, 16):
            G.step(i)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert np.isfinite(G.histories()["loss"]).all()


def test_end_to_end_on_the_box_room_with_the_median_depth(room):
    """test_gpu_gs_train's end-to-end recipe with depth_type=1: held-out PSNR and the mesh of the jointly trained SDF. Measured on an
    H100: see DESIGN 7o."""
    import test_gpu_gs_train as GS
    from gssdf_b200 import mesh as ME
    from gssdf_b200 import metrics as MT
    from gssdf_b200 import scene as S
    S_ = GS._sdf_trainer(room, 200, seed=5, outlier_remove=True)
    c2w = GS._poses(72, 9)
    imgs = GS._images(c2w)
    train, test = slice(0, 60), slice(60, 72)
    G = GS._gs_trainer(room, S_, (c2w[train].contiguous(), imgs[train].contiguous()), 2000, sh_degree=1, capacity_mult=32,
                       outlier_remove=True, refine_gs_struct_start_iter=1000, densify=dict(refine_start_iter=200, refine_every=100),
                       sh_degree_interval=500, depth_type=1)
    G.run()
    h = G.histories()
    st = G.state()
    vms = torch.linalg.inv(c2w[test].to(torch.float64)).to(torch.float32)
    renders = torch.stack([st["render"](vm) for vm in vms])
    full, _ = MT.eval_render(renders.clamp(0, 1), imgs[test], [f"{i}.png" for i in range(12)])
    v, f, _ = ME.meshing(room["tree"], st["net"], room["margin"][0], room["margin"][1], 0.025)
    gt = S.box_wall_points(0.01)
    mm = ME.eval_mesh(v, f, torch.from_numpy(gt).to(_dev()), mesh_sample_point=1_000_000, gt_bbx_mask_on=False)
    print(f"depth_type 1: held-out {full}; mesh {mm}; N_live {h['n_live'][-1]}; loss last {h['loss'][-3:]}")
    assert full["PSNR"] > 24.0
    assert mm["MAE_accuracy (cm)"] < 1.0 and mm["MAE_completeness (cm)"] < 1.0 and mm["F-score (%)"] > 97.0
