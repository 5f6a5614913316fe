"""f-6 splat initialisation on the CPU: the fp32 restatement of the epilogue (tests/gs_init_oracle.py) against fp64, the splat frame
against the SDF normal, the quirks of the crafted cases, the reference's stride / sky / NaN-filter rules restated literally, and the
C ABI's argument checks (no launch)."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

import gs_init_oracle as GO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32


def _quadratic_field(n, delta, seed=0):
    """SDF values at a point and its six offsets from s(x + d) = s0 + g.d + d.H.d / 2 (diagonal H), fp32; plus y1."""
    rng = np.random.default_rng(seed)
    s0 = rng.uniform(-0.1, 0.1, n)
    g = rng.normal(size=(n, 3))
    g /= np.linalg.norm(g, axis=1, keepdims=True)
    h = rng.normal(scale=10.0, size=(n, 3))
    s7 = np.empty((7, n))
    s7[0] = s0
    for k in range(3):
        s7[1 + 2 * k] = s0 + g[:, k] * delta + 0.5 * h[:, k] * delta ** 2
        s7[2 + 2 * k] = s0 - g[:, k] * delta + 0.5 * h[:, k] * delta ** 2
    return s7.astype(f32), rng.normal(scale=0.05, size=n).astype(f32)


def test_epilogue_fp32_agrees_with_fp64_on_well_conditioned_rows():
    delta = float(f32(0.025))
    s7, y1 = _quadratic_field(20000, delta)
    a = GO.epilogue(s7, y1, delta, 10.0, np.float32)
    b = GO.epilogue(s7, y1, delta, 10.0, np.float64)
    ok = GO.well_conditioned(b["trace"])
    assert ok.mean() > 0.9
    np.testing.assert_allclose(a["grad"], b["grad"], rtol=1e-6, atol=1e-6)
    # (s+ + s-) - 2 s cancels: |error| <= 3 ulp(0.1) * fl(1/delta^2)
    np.testing.assert_allclose(a["curv_dom"], b["curv_dom"], rtol=0, atol=3 * 7.5e-9 * 1600 * 1.01)
    np.testing.assert_allclose(a["opacity"], b["opacity"], rtol=1e-6)
    err = np.abs(a["quaternion"][ok] - b["quaternion"][ok]).max()
    print(f"fp32 vs fp64 quaternion on {int(ok.sum())} well-conditioned rows: max |diff| {err:.2e}")
    assert err < 1e-4


def test_splat_z_axis_is_the_sdf_normal():
    """Column 2 of R(q) is normalize(grad): the permutation [b2, b3, b1] puts the SDF normal on the splat's z axis."""
    delta = float(f32(0.025))
    s7, y1 = _quadratic_field(20000, delta, seed=1)
    r = GO.epilogue(s7, y1, delta, 10.0, np.float32)
    ok = GO.well_conditioned(r["trace"])
    R = GO.quat_to_matrix(r["quaternion"][ok])
    n = r["grad"][ok].astype(np.float64)
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    # fp32 accuracy of the axis-angle round trip: the axis carries ~1e-7 / sin(angle), and sin(angle) >= 0.1 on these rows
    assert np.abs(R[:, :, 2] - n).max() < 5e-5
    assert np.abs(np.linalg.norm(r["quaternion"][ok].astype(np.float64), axis=1) - 1).max() < 1e-6


def test_crafted_cases_give_the_documented_quirks():
    a1, a2, names = GO.crafted_cases()
    q, trace = GO.rot6d_to_quat(a1, a2)
    byname = {}
    for i, nm in enumerate(names):
        byname.setdefault(nm, []).append(i)
    # angle 0: the axis is 0 / 0 = NaN -> nan_to_num -> 0, and q = (1, 0, 0, 0)
    assert np.array_equal(q[byname["identity"][0]], [1, 0, 0, 0])
    # exact half-turns: acos(-1) = pi in fp32, the axis numerators are exactly 0 -> axis 0, q = (cos(pi_f / 2), 0, 0, 0) ~ (-4.4e-8, 0, 0, 0)
    for nm in ("half-turn x", "half-turn y", "half-turn z"):
        i = byname[nm][0]
        assert trace[i] == -1 and np.array_equal(q[i][1:], [0, 0, 0]) and abs(q[i][0]) < 1e-7, (nm, q[i])
    # a1 parallel to a2: b2 = b3 = 0, trace = b1[2], q = (cos(angle / 2), 0, 0, 0) is not a unit quaternion
    i = byname["parallel"][0]
    assert np.array_equal(q[i][1:], [0, 0, 0]) and abs(q[i][0] - np.cos(np.pi / 4)) < 1e-6
    assert np.isfinite(q).all()
    # zero vectors: normalize gives 0 (eps 1e-12), never NaN
    for nm in ("zero a1", "zero a2", "zero both"):
        assert np.isfinite(q[byname[nm][0]]).all()
    # near identity: the fp32 trace lands on 3 and q = (1, 0, 0, 0) up to the rounding of the tiny angle
    near = byname["near identity"]
    assert (np.abs(q[near][:, 0] - 1) < 1e-6).all() and (np.abs(q[near][:, 1:]) < 1e-3).all()
    # an fp32 trace past 3 (a matrix whose diagonal rounds above 1) makes acos NaN: the whole quaternion becomes 0
    u = f32(1.000001)
    qm, tm = GO.matrix_to_quat(np.diag([f32(1), u, u]).astype(f32)[None], np.float32)
    assert tm[0] > 3 and np.array_equal(qm[0], np.zeros(4, np.float32))


@pytest.mark.parametrize("n,cap", [(10, 20), (20, 20), (21, 20), (39, 20), (40, 20), (41, 20), (1000, 7), (123457, 10000)])
def test_stride_rule_matches_the_reference_slice(n, cap):
    from gssdf_b200 import gs_init
    got = list(gs_init.anchor_indices(n, cap))
    assert got == GO.anchor_indices_reference(n, cap)
    if n > cap:
        assert n - 1 not in got  # slice(0, 0, -1, step) stops before the last vertex


@pytest.mark.parametrize("spatial_scale,inner", [(1.0, 14.0), (0.3, 5.0), (1.7, 20.0), (2.3, 8.0), (0.001, 14.0)])
def test_sky_count_and_scale(spatial_scale, inner):
    from gssdf_b200 import gs_init
    n, r, s = GO.sky_reference(spatial_scale, inner)
    assert gs_init.sky_count(spatial_scale) == n
    assert gs_init.sky_radius(inner) == r
    if n > 0:
        assert gs_init.sky_log_scale(inner, n) == s
    # torch::full(log(mesh_res)) of the anchors: an fp32 value of the double log
    assert gs_init.anchor_log_scale(0.025) == float(f32(np.log(np.float64(f32(0.025)))))


def test_nan_filter_follows_the_reference_order():
    """features_dc is drawn for all rows before the filter; isnan only (+inf opacities pass); the same rows go in every tensor."""
    from gssdf_b200 import gs_init
    n = 12
    g = torch.Generator().manual_seed(4)
    anchors, scaling = torch.randn(n, 3, generator=g), torch.randn(n, 3, generator=g)
    quat, opa = torch.randn(n, 4, generator=g), torch.randn(n, generator=g)
    anchors[1, 0] = float("nan"); scaling[4, 2] = float("nan"); quat[7, 3] = float("nan"); opa[9] = float("nan")
    opa[10] = float("inf"); anchors[11, 1] = float("inf")
    out, num_nan = gs_init.finish_rows(anchors, scaling, quat, opa, 2, torch.Generator().manual_seed(8))
    # literal restatement of neural_gaussian.cpp:403-424
    dc = torch.rand(n, 1, 3, generator=torch.Generator().manual_seed(8))
    is_nan = anchors.isnan().any(-1) | scaling.isnan().any(-1) | quat.isnan().any(-1) | opa.isnan()
    valid = (~is_nan).nonzero().squeeze()
    assert num_nan == 4 == int(is_nan.sum())
    for k, t in (("anchors", anchors), ("scaling", scaling), ("quaternion", quat), ("opacity", opa), ("features_dc", dc)):
        assert torch.equal(out[k], t.index_select(0, valid)), k
    assert out["features_rest"].shape == (8, 8, 3) and out["offsets"].shape == (8, 3)
    assert float(out["opacity"][-2]) == float("inf")


def _args(name, **kw):
    from gssdf_b200 import _lib
    return _lib.make_args(name, **kw)


def test_cabi_exports_and_rejects_without_launch():
    from gssdf_b200 import _lib
    L = _lib.lib()
    for sym in ("gssdf_sdf_init_gs", "gssdf_sdf_init_gs_workspace_bytes", "gssdf_rot6d_to_quat"):
        assert sym in _lib.FUNCS and hasattr(L, sym)
    assert L.gssdf_sdf_init_gs_workspace_bytes(1000) >= 56 * 1000
    assert L.gssdf_sdf_init_gs_workspace_bytes(-1) == 0

    def call(**over):
        kw = dict(n=100, x=0x1000, delta=0.025, bce_isigma=10.0, quaternion=0x2000, workspace=0x3000,
                  workspace_bytes=L.gssdf_sdf_init_gs_workspace_bytes(100))
        kw.update(over)
        a = _args("gssdf_sdf_init_gs_args", **kw)
        a.net.table_half, a.net.mlp = 0x8000, 0x9000
        rc = L.gssdf_sdf_init_gs(C.byref(a), None)
        return rc, L.gssdf_last_error().decode()

    rc, msg = call(n=-1)
    assert rc == -1 and "n must" in msg
    for d in (0.0, -0.025, float("nan"), float("inf")):
        rc, msg = call(delta=d)
        assert rc == -1 and "delta" in msg
    rc, msg = call(quaternion=None)
    assert rc == -1 and "quaternion" in msg
    rc, msg = call(workspace_bytes=L.gssdf_sdf_init_gs_workspace_bytes(100) - 1)
    assert rc == -1 and "workspace" in msg
    assert call(n=0, x=None, workspace=None, workspace_bytes=0)[0] == 0  # empty input: a legal no-op

    def call_q(**over):
        kw = dict(n=100, a1=0x1000, a2=0x2000, quaternion=0x3000)
        kw.update(over)
        a = _args("gssdf_rot6d_to_quat_args", **kw)
        return L.gssdf_rot6d_to_quat(C.byref(a), None), L.gssdf_last_error().decode()

    assert call_q(n=-5)[0] == -1
    rc, msg = call_q(quaternion=None)
    assert rc == -1 and "quaternion" in msg
    assert call_q(n=0, a1=None, a2=None)[0] == 0


def test_shim_entry_point_is_built():
    so = os.path.join(ROOT, "gs-sdf_b200", "gssdf_shim.so")
    assert os.path.exists(so), "gssdf_shim.so is built by build()"
    nm = shutil.which("nm")
    if nm is None:
        pytest.skip("needs binutils' nm")
    out = subprocess.run([nm, "-DC", "--defined-only", so], capture_output=True, text=True, check=True).stdout
    assert ("gssdf::init_gs_with_sdf[abi:cxx11](TCNNEncoding const&, torch::nn::Sequential&, at::Tensor const&, float, float, "
            "at::Tensor const&, float, bool)") in out
