"""The fp64 arbiter of the splat VJP kernels (tests/splat_vjp_oracle.py) on the CPU: its raw-parameter chain rule against float64
torch autograd, its agreement with the reference CUDA goldens, and -- for every scene the GPU tests use -- proof that each branch
they compare shows up at their tolerance, so that dropping it, flipping its sign or losing one of its factors would fail them."""
import os

import numpy as np
import pytest

import splat_vjp_oracle as A
import splat_vjp_scenes as SC
from gssdf_b200 import scene as S

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _small_raw(seed=3, N=400, K=16):
    rng = np.random.default_rng(seed)
    sc = SC.scene("edge")
    raw = {k: v[:N].copy() for k, v in sc["raw"].items()}
    sh = rng.normal(-1.0, 1.5, (N, K, 3)).astype(np.float32)
    raw.update(dc=np.ascontiguousarray(sh[:, :1]), rest=np.ascontiguousarray(sh[:, 1:]))
    return sc, raw


def _fw(O, sc, means, scales, N):
    p = O.project2dgs_fwd(means, sc["quats"][:N], scales, sc["V"], sc["K"], sc["W"], sc["H"], S.NEAR, S.FAR, 0.0, None, "f32")
    assert p["nnz"] > 50
    cot, rn = SC.cotangents(p["nnz"])
    return dict(camera_ids=p["camera_ids"], gaussian_ids=p["gaussian_ids"], ray_transforms=p["ray_transforms"], randns=rn,
                radii=p["radii"]), cot


def test_chain_rule_matches_float64_autograd(oracle):
    """Raw layout of the arbiter == float64 torch autograd of add / exp / sigmoid / cat applied to its activated-layout result."""
    torch = pytest.importorskip("torch")
    sc, raw = _small_raw()
    N, deg = len(raw["anchors"]), 3
    means, scales, opac = A.activate(raw)
    act = dict(means=means, scales=scales, opacities=opac, sh=np.concatenate([raw["dc"], raw["rest"]], 1))
    fw, cot = _fw(oracle, sc, means, scales, N)
    vc = np.random.default_rng(8).standard_normal((len(fw["gaussian_ids"]), 3)).astype(np.float32)
    pa, pr = A.project_bwd(oracle, act, sc["quats"][:N], sc["V"], sc["K"], fw, cot), \
        A.project_bwd(oracle, raw, sc["quats"][:N], sc["V"], sc["K"], fw, cot)
    ca, cr = A.colors_bwd(oracle, act, sc["V"], fw, vc, deg), A.colors_bwd(oracle, raw, sc["V"], fw, vc, deg)
    assert np.abs(pa["v_scales"]).max() > 0 and np.abs(ca["v_means"]).max() > 0 and np.abs(pa["v_opacities"]).max() > 0
    L = {k: torch.tensor(np.asarray(v, np.float64), requires_grad=True) for k, v in raw.items()}
    m = L["anchors"] + L["offsets"]
    loss = (m * torch.from_numpy(pa["v_means"] + ca["v_means"])).sum() + (torch.exp(L["log_scales"]) * torch.from_numpy(pa["v_scales"])).sum() \
        + (torch.sigmoid(L["logits"]) * torch.from_numpy(pa["v_opacities"])).sum() \
        + (torch.cat([L["dc"], L["rest"]], 1) * torch.from_numpy(ca["v_sh"])).sum()
    loss.backward()
    g = {k: v.grad.numpy() for k, v in L.items()}
    close = lambda a, b: np.testing.assert_allclose(a, b, rtol=1e-6, atol=1e-12 * max(np.abs(b).max(), 1e-300))
    close(pr["v_means"] + cr["v_means"], g["offsets"])
    close(pr["v_means"] + cr["v_means"], g["anchors"])
    close(pr["v_scales"], g["log_scales"])
    assert (pr["v_scales"][:, 2] == 0).all()
    close(pr["v_opacities"], g["logits"])
    close(cr["v_dc"], g["dc"])
    close(cr["v_rest"], g["rest"])
    np.testing.assert_array_equal(pr["v_quats"], pa["v_quats"])


def test_raw_layout_equals_activated_oracle_call(oracle):
    """The raw-layout arbiter is the plain fp64 oracle call on the activated scene, times the activation derivatives."""
    sc, raw = _small_raw(seed=4)
    N, deg = len(raw["anchors"]), 2
    means, scales, opac = A.activate(raw)
    fw, cot = _fw(oracle, sc, means, scales, N)
    gid = fw["gaussian_ids"]
    d = oracle.project2dgs_bwd(means, sc["quats"][:N], scales, sc["V"], sc["K"], fw["camera_ids"], gid, fw["ray_transforms"], fw["randns"],
                               cot["v_means2d"], cot["v_depths"], cot["v_ray_transforms"], cot["v_normals"], cot["v_samples"], "f64")
    r = A.project_bwd(oracle, raw, sc["quats"][:N], sc["V"], sc["K"], fw, cot)
    np.testing.assert_array_equal(r["v_means"], d["v_means"])
    np.testing.assert_array_equal(r["v_quats"], d["v_quats"])
    np.testing.assert_array_equal(r["v_scales"][:, :2], d["v_scales"][:, :2] * scales[:, :2])
    o = opac.astype(np.float64)[gid]
    vo = np.zeros(N)
    np.add.at(vo, gid, cot["v_pt_opacities"] * o * (1 - o))
    np.testing.assert_allclose(r["v_opacities"], vo, rtol=1e-6, atol=0)  # fp64 sigmoid vs its float32 rounding
    vc = np.random.default_rng(9).standard_normal((len(gid), 3)).astype(np.float32)
    sh = np.concatenate([raw["dc"], raw["rest"]], 1)
    col, dirs = oracle.view_colors_fwd(sc["V"], means, fw["radii"], sh, fw["camera_ids"], gid, deg, "f64")
    vcoef, vdir = oracle.sh_bwd(deg, dirs, sh[gid], vc * (col > 0), None, "f64")
    c = A.colors_bwd(oracle, raw, sc["V"], fw, vc, deg)
    np.testing.assert_array_equal(c["v_sh"][gid], vcoef)
    np.testing.assert_array_equal(c["v_means"][gid], vdir)
    assert (c["v_rest"][:, (deg + 1) ** 2 - 1:] == 0).all()  # bases above the active degree
    outside = np.setdiff1d(np.arange(N), gid)
    assert len(outside) and (c["v_sh"][outside] == 0).all() and (c["v_means"][outside] == 0).all()


@pytest.mark.parametrize("name", ["a", "b"])
def test_arbiter_reproduces_reference_cuda_goldens(oracle, name):
    """Fed the goldens' own forward state and cotangents, the arbiter reproduces the reference kernels' v_means / v_quats / v_scales /
    v_coeffs / v_dirs within the bounds ref_cuda_checks.check_file uses."""
    from helpers import assert_close_frac
    from ref_cuda_checks import rel_l2, scene_of
    d = np.load(os.path.join(GOLDEN, f"ref_cuda_{name}.npz"))
    sc, V, K, N, W, H, deg = scene_of(d)
    gid = d["gaussian_ids"]
    nnz = len(gid)
    fw = dict(camera_ids=d["camera_ids"], gaussian_ids=gid, ray_transforms=d["ray_transforms"], randns=S.randns(N)[:nnz], radii=d["radii"])
    cot = dict(v_means2d=d["v_means2d"], v_ray_transforms=d["v_ray_transforms"], v_normals=d["v_normals"], v_samples=d["v_samples"])
    pb = A.project_bwd(oracle, sc, sc["quats"], V, K, fw, cot)
    for k in ("v_means", "v_quats", "v_scales"):
        assert rel_l2(pb[k], d[k]) < 5e-4, f"{k}: {rel_l2(pb[k], d[k]):.2e}"
    c = A.colors_bwd(oracle, sc, V, fw, d["v_colors"], deg, colors=d["colors"])
    assert_close_frac(c["v_sh"][gid], d["v_coeffs"], 1e-4, 1e-6 * np.abs(d["v_coeffs"]).max(), 0.0, "v_coeffs")
    if deg > 0:
        assert_close_frac(c["v_means"][gid], d["v_dirs"], 2e-4, 1e-5 * np.abs(d["v_dirs"]).max(), 0.0, "v_dirs")


def _visible(O, sc):
    act = sc["act"]
    p = O.project2dgs_fwd(act["means"], sc["quats"], act["scales"], sc["V"], sc["K"], sc["W"], sc["H"], S.NEAR, S.FAR, 0.0, None, "f32")
    rows = np.zeros(sc["N"], bool)
    rows[p["gaussian_ids"]] = True
    return p, rows


def _frac_out(got, ref, rows):
    """Largest fraction of compared entries outside the GPU tolerance over the compared gradients."""
    return max(A.tol_bad(got[k], ref[k], rows=rows)[0].mean() for k in ref)


def _rows(sc, gid, excluded):
    rows = np.zeros(sc["N"], bool)
    rows[gid[~excluded]] = True
    return rows


@pytest.mark.parametrize("mode", ["act", "raw"])
@pytest.mark.parametrize("name", list(SC.SCENES))
def test_projection_branches_visible_at_gpu_tolerance(oracle, name, mode):
    """For each cotangent branch: in its own call, and in the call with all six (SC.ALL_WEIGHTS), the branch removed or its sign flipped
    puts >= 5 % of the compared entries of some gradient outside rtol 1e-4 / atol 1e-6 max|ref|. So do r0 <-> r1 swapped in the sample
    term and, in the raw layout, the s factor of d/d log s or the sigmoid' of d/d logit dropped. The conditioning rules exclude at most
    SC.MAX_EXCLUDED of the rows."""
    sc = SC.scene(name)
    p, _ = _visible(oracle, sc)
    gid = p["gaussian_ids"]
    cot, rn = SC.cotangents(p["nnz"])
    ex = SC.exclusions(sc, p)
    print(f"{name}: {p['nnz']} visible, excluded " + ", ".join(f"{b} {int(m.sum())}" for b, m in ex.items() if m.any()))
    assert ex["all"].mean() <= SC.MAX_EXCLUDED
    fw = dict(camera_ids=p["camera_ids"], gaussian_ids=gid, ray_transforms=p["ray_transforms"], randns=rn)
    params = sc[mode]
    bwd = lambda c, f=fw: A.project_bwd(oracle, params, sc["quats"], sc["V"], sc["K"], f, c)
    w_cot = {b: (SC.ALL_WEIGHTS[b] * cot[b]).astype(np.float32) for b in A.BRANCHES}
    full = bwd(w_cot)
    rows_all = _rows(sc, gid, ex["all"])
    lin = lambda a, b, s: {k: a[k] + s * b[k] for k in a}
    for b in A.BRANCHES:
        one, rows = bwd({b: cot[b]}), _rows(sc, gid, ex[b])
        w_one = bwd({b: w_cot[b]})
        zero = {k: np.zeros_like(v) for k, v in one.items()}
        fr = dict(removed=_frac_out(zero, one, rows), flipped=_frac_out(lin(zero, one, -1), one, rows),
                  removed_all=_frac_out(lin(full, w_one, -1), full, rows_all), flipped_all=_frac_out(lin(full, w_one, -2), full, rows_all))
        print(f"  {mode} {b}: " + ", ".join(f"{k} {v:.3f}" for k, v in fr.items()))
        assert min(fr.values()) >= 0.05, (b, fr)
    one = bwd({"v_samples": cot["v_samples"]})
    swapped = bwd({"v_samples": cot["v_samples"]}, dict(fw, randns=np.ascontiguousarray(rn[:, ::-1])))
    assert _frac_out(swapped, one, _rows(sc, gid, ex["v_samples"])) >= 0.05
    if mode == "raw":
        s = sc["act"]["scales"].astype(np.float64)
        o = sc["act"]["opacities"].astype(np.float64)
        no_s = dict(full, v_scales=full["v_scales"] / s)
        no_sig = dict(full, v_opacities=full["v_opacities"] / (o * (1 - o)))
        assert _frac_out(no_s, full, rows_all) >= 0.05 and _frac_out(no_sig, full, rows_all) >= 0.05


SH_CASES = [(16, 0, True), (16, 1, True), (16, 2, True), (16, 3, True), (25, 4, True), (16, 1, False)]  # (K, degree, split dc/rest)


@pytest.mark.parametrize("K,deg,split", SH_CASES)
def test_sh_clamp_and_direction_terms_visible_at_gpu_tolerance(oracle, K, deg, split):
    """The SH scene clamps 20 %..80 % of the (splat, channel) colours, and dropping the clamp mask puts >= 5 % of the visible v_dc
    (v_sh) entries outside the GPU tolerance; at degree >= 1 the view-direction gradient v_means is non-zero on every visible splat with an unclamped channel."""
    sc = SC.scene("box")
    p, rows = _visible(oracle, sc)
    shs = SC.sh_scene("box", K)
    params = dict(sc["raw"], dc=shs["dc"], rest=shs["rest"]) if split else dict(sc["act"], sh=shs["sh"])
    fw = dict(camera_ids=p["camera_ids"], gaussian_ids=p["gaussian_ids"], radii=p["radii"])
    vc = np.random.default_rng(41).standard_normal((p["nnz"], 3)).astype(np.float32)
    ref = A.colors_bwd(oracle, params, sc["V"], fw, vc, deg)
    clamped = 1 - ref["mask"].mean()
    print(f"K {K} degree {deg} split {split}: {clamped:.3f} of the colours clamp")
    assert 0.2 <= clamped <= 0.8
    nomask = A.colors_bwd(oracle, params, sc["V"], fw, vc, deg, colors=np.ones_like(vc))
    assert A.tol_bad(nomask["v_dc"], ref["v_dc"], rows=rows)[0].mean() >= 0.05
    if deg > 0:
        lit = np.zeros(sc["N"], bool)
        lit[p["gaussian_ids"][ref["mask"].any(1)]] = True
        assert (np.abs(ref["v_means"][lit]).max(1) > 0).all()
        assert A.tol_bad(nomask["v_means"], ref["v_means"], rows=rows)[0].mean() >= 0.05
