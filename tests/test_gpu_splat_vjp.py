"""The two per-splat VJP kernels against the fp64 arbiter (tests/splat_vjp_oracle.py), one cotangent branch at a time, in the layout the
trainer runs them: raw parameters (anchors + offsets, log-scales, logits), SH split into features_dc / features_rest at every active
degree, capacity-sized buffers whose rows at or beyond nnz hold NaN.

The GPU forward runs once per scene; its own outputs (camera_ids, gaussian_ids, radii, ray_transforms, pt_opacities, colours) feed both
the kernel backward and the arbiter, so only the backward is judged. Bar: rtol 1e-4 with atol 1e-6 x max|ref| of the branch under test,
no bad-entry fraction; rows leave the comparison only by the fp64 conditioning rules of splat_vjp_scenes.exclusions, counted and bounded.
tests/test_splat_vjp_host.py proves on the CPU that every branch compared here moves >= 5 % of some gradient's entries at this bar."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import splat_vjp_oracle as A  # noqa: E402
import splat_vjp_scenes as SC  # noqa: E402
from gssdf_b200 import scene as S  # noqa: E402

RTOL, ATOL_REL = 1e-4, 1e-6


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _np(t):
    return t.detach().cpu().numpy()


def _cap_buf(rows, cap, dev, fill=float("nan")):
    """A capacity-sized buffer: `rows` in front, `fill` behind (what the trainer's torch.empty buffers may hold)."""
    rows = np.asarray(rows)
    out = torch.full((cap,) + rows.shape[1:], fill, dtype=torch.float32, device=dev)
    out[:len(rows)] = _t(rows.astype(np.float32), dev)
    return out


def _forward(O, sc, mode, dev):
    """GPU projection forward of the scene (C = 1, cap = N); checks the visible set against the f32 oracle and returns the packed
    outputs with every float row at or beyond nnz set to NaN and the id rows pointing at an invisible splat."""
    from gssdf_b200 import cabi
    N, cap = sc["N"], sc["N"]
    e = lambda *s, dt=torch.float32: torch.empty(*s, dtype=dt, device=dev)
    out = dict(camera_ids=e(cap, dt=torch.int64), gaussian_ids=e(cap, dt=torch.int64), radii=e(cap, 2, dt=torch.int32), means2d=e(cap, 2),
               depths=e(cap), ray_transforms=e(cap, 3, 3), normals=e(cap, 3), samples=e(cap, 3), sample_weights=e(cap, 1), pt_opacities=e(cap),
               indptr=e(2, dt=torch.int32))
    counts, ws = cabi.new_counts(dev), cabi.Workspace(dev)
    t = {k: _t(v, dev) for k, v in sc[mode].items()}
    raw = mode == "raw"
    cabi.project2dgs_fwd(t["anchors" if raw else "means"], _t(sc["quats"], dev), t["log_scales" if raw else "scales"], _t(sc["V"], dev),
                         _t(sc["K"], dev), sc["W"], sc["H"], S.NEAR, S.FAR, 0.0, None, cap, out, counts, ws,
                         opacities=t["logits" if raw else "opacities"], mean_offsets=t["offsets"] if raw else None, raw_params=raw)
    torch.cuda.synchronize()
    nnz = int(counts[cabi.NNZ])
    act = sc["act"]
    p32 = O.project2dgs_fwd(act["means"], sc["quats"], act["scales"], sc["V"], sc["K"], sc["W"], sc["H"], S.NEAR, S.FAR, 0.0, None, "f32")
    gid = _np(out["gaussian_ids"][:nnz])
    assert nnz == p32["nnz"] and np.array_equal(gid, p32["gaussian_ids"]), "visible set differs from the f32 oracle"
    ghost = int(np.setdiff1d(np.arange(N), gid)[0])
    for k in ("means2d", "depths", "ray_transforms", "normals", "pt_opacities"):
        out[k][nnz:] = float("nan")
    out["gaussian_ids"][nnz:] = ghost
    out["camera_ids"][nnz:] = 0
    out["radii"][nnz:] = 1
    p = {k: _np(out[k][:nnz]) for k in ("camera_ids", "gaussian_ids", "radii", "means2d", "ray_transforms", "pt_opacities")}
    p["nnz"] = nnz
    return out, counts, p, ghost


def _params_gpu(sc, mode, dev):
    t = {k: _t(v, dev) for k, v in sc[mode].items()}
    if mode == "raw":
        return dict(means=t["anchors"], scales=t["log_scales"], offsets=t["offsets"], raw=True)
    return dict(means=t["means"], scales=t["scales"], offsets=None, raw=False)


def _check(name, got, ref, rows, label):
    """rtol 1e-4, atol 1e-6 max|ref| on `rows`; no NaN anywhere; rows outside the visible set bit-exactly 0."""
    bad, rel = A.tol_bad(got, ref, RTOL, ATOL_REL, rows=rows)
    assert not np.isnan(got).any(), f"{label} {name}: NaN"
    assert not bad.any(), f"{label} {name}: {int(bad.sum())} of {bad.size} entries off, max err/(|ref| + atol) {rel:.2e}"
    return rel


@pytest.mark.parametrize("mode", ["act", "raw"])
@pytest.mark.parametrize("name", list(SC.SCENES))
def test_projection_bwd_one_branch_at_a_time(oracle, name, mode):
    """Six calls with one cotangent branch each, then one with all six (SC.ALL_WEIGHTS); v_means / v_quats / v_scales / v_opacities
    against the arbiter, activated (raw_params=0) and in the trainer's raw layout (raw_params=1, mean_offsets, the forward's pt_opacities)."""
    from gssdf_b200 import cabi
    dev = _dev()
    sc = SC.scene(name)
    N = sc["N"]
    out, counts, p, ghost = _forward(oracle, sc, mode, dev)
    nnz, gid = p["nnz"], p["gaussian_ids"]
    cot, rn = SC.cotangents(nnz)
    ex = SC.exclusions(sc, p)
    assert ex["all"].mean() <= SC.MAX_EXCLUDED
    visible = np.zeros(N, bool)
    visible[gid] = True
    prm = _params_gpu(sc, mode, dev)
    quats, V, K = _t(sc["quats"], dev), _t(sc["V"], dev), _t(sc["K"], dev)
    randns = _cap_buf(rn, N, dev)
    fw = dict(camera_ids=p["camera_ids"], gaussian_ids=gid, ray_transforms=p["ray_transforms"], randns=rn,
              pt_opacities=p["pt_opacities"] if mode == "raw" else None)
    cases = [(b, {b: cot[b]}) for b in A.BRANCHES]
    cases.append(("all", {b: (SC.ALL_WEIGHTS[b] * cot[b]).astype(np.float32) for b in A.BRANCHES}))
    for label, c in cases:
        g = {b: _cap_buf(c[b], N, dev) if b in c else None for b in A.BRANCHES}
        res = dict(v_means=torch.zeros(N, 3, device=dev), v_quats=torch.zeros(N, 4, device=dev), v_scales=torch.zeros(N, 3, device=dev),
                   v_opacities=torch.zeros(N, device=dev))
        cabi.project2dgs_bwd(prm["means"], quats, prm["scales"], V, K, sc["W"], sc["H"], N, counts, out["camera_ids"], out["gaussian_ids"],
                             out["ray_transforms"], randns, g["v_means2d"], g["v_depths"], g["v_ray_transforms"], g["v_normals"],
                             g["v_samples"], res["v_means"], res["v_quats"], res["v_scales"], v_pt_opacities=g["v_pt_opacities"],
                             v_opacities=res["v_opacities"], mean_offsets=prm["offsets"], raw_params=prm["raw"],
                             pt_opacities=out["pt_opacities"])
        torch.cuda.synchronize()
        ref = A.project_bwd(oracle, sc[mode], sc["quats"], sc["V"], sc["K"], fw, c)
        rows = np.ones(N, bool)
        rows[gid[ex[label]]] = False
        rels = []
        for k, v in res.items():
            got = _np(v)
            rels.append(f"{k} {_check(k, got, ref[k], rows, f'{name} {mode} {label}'):.1e}")
            assert (got[~visible] == 0).all() and (got[ghost] == 0).all(), f"{label} {k}: rows outside gaussian_ids touched"
        if prm["raw"]:
            assert (_np(res["v_scales"])[:, 2] == 0).all()
        print(f"{name} {mode} {label}: excluded {int(ex[label].sum())} of {nnz} rows; max err/(|ref| + atol): " + ", ".join(rels))


@pytest.mark.parametrize("K,deg,split", [(16, 0, True), (16, 1, True), (16, 2, True), (16, 3, True), (25, 4, True), (16, 1, False)])
def test_view_colors_bwd_trainer_layout(oracle, K, deg, split):
    """view_colors fwd / bwd with 20 %..80 % of the colours clamped: split features_dc / features_rest with mean_offsets (the trainer)
    at active degrees 0..4, and one unsplit [N,16,3] call at degree 1 (coefficient stride K > (deg+1)^2). Colours, v_dc, v_rest and
    v_offsets against the arbiter; v_rest rows of inactive bases and rows of splats outside gaussian_ids bit-exactly 0."""
    from gssdf_b200 import cabi
    dev = _dev()
    sc = SC.scene("box")
    N = sc["N"]
    mode = "raw" if split else "act"
    out, counts, p, ghost = _forward(oracle, sc, mode, dev)
    nnz, gid = p["nnz"], p["gaussian_ids"]
    shs = SC.sh_scene("box", K)
    params = dict(sc["raw"], dc=shs["dc"], rest=shs["rest"]) if split else dict(sc["act"], sh=shs["sh"])
    prm = _params_gpu(sc, mode, dev)
    V = _t(sc["V"], dev)
    sh, rest = (_t(shs["dc"], dev), _t(shs["rest"], dev)) if split else (_t(shs["sh"], dev), None)
    colors = torch.full((N, 3), float("nan"), device=dev)
    cabi.view_colors_fwd(V, prm["means"], sh, deg, N, counts, out["camera_ids"], out["gaussian_ids"], out["radii"], colors,
                         mean_offsets=prm["offsets"], sh_rest=rest)
    vc = np.random.default_rng(41).standard_normal((nnz, 3)).astype(np.float32)
    v_colors = _cap_buf(vc, N, dev)
    v_sh = torch.zeros(N, 1 if split else K, 3, device=dev)
    v_rest = torch.zeros(N, K - 1, 3, device=dev) if split else None
    v_means = torch.zeros(N, 3, device=dev)
    cabi.view_colors_bwd(V, prm["means"], sh, deg, N, counts, out["camera_ids"], out["gaussian_ids"], out["radii"], colors, v_colors,
                         v_sh, v_means, mean_offsets=prm["offsets"], sh_rest=rest, v_sh_rest=v_rest)
    torch.cuda.synchronize()
    col = _np(colors[:nnz])
    ref = A.colors_bwd(oracle, params, sc["V"], dict(p), vc, deg, colors=col)
    from helpers import assert_close_frac
    assert_close_frac(col, ref["colors"], 1e-4, 1e-5, 0.0, "colors")
    clamped = float((col == 0).mean())
    assert 0.2 <= clamped <= 0.8, clamped
    got = dict(v_dc=_np(v_sh[:, :1]), v_rest=_np(v_rest) if split else _np(v_sh[:, 1:]), v_offsets=_np(v_means))
    want = dict(v_dc=ref["v_dc"], v_rest=ref["v_rest"], v_offsets=ref["v_means"])
    outside = np.ones(N, bool)
    outside[gid] = False
    rels = []
    for k in got:
        rels.append(f"{k} {_check(k, got[k], want[k], None, f'K {K} degree {deg}'):.1e}")
        assert (got[k][outside] == 0).all() and (got[k][ghost] == 0).all(), f"{k}: rows outside gaussian_ids touched"
    assert (got["v_rest"][:, (deg + 1) ** 2 - 1:] == 0).all(), "v_rest of inactive bases"
    if not split:
        assert (_np(v_sh)[:, (deg + 1) ** 2:] == 0).all()
    if deg > 0:
        assert np.abs(got["v_offsets"]).max() > 0
    print(f"K {K} degree {deg} split {split}: {clamped:.3f} of the colours clamp; max err/(|ref| + atol): " + ", ".join(rels))
