"""f-10 on the CPU: the numpy restatement of gssdf_knn3_mean_dist2 (tests/knn_oracle.py) against a brute-force replay of simple-knn's
updateKBest and against exact rational arithmetic, the small-cloud and non-finite rules, gs_init's random_quat and init_point_indices
against the reference's statements, and the C ABI's argument checks (no launch)."""
import ctypes as C
import math
from fractions import Fraction

import numpy as np
import pytest
import torch

import knn_oracle as KO

f32 = np.float32


def test_fma_emulation_rounds_once():
    """fma32 against exact rationals, on random values and on products that land exactly on fp32 midpoints of the addend."""
    rng = np.random.default_rng(0)
    a = rng.standard_normal(2000).astype(f32)
    c = (rng.standard_normal(2000) * 4).astype(f32)
    a[:500] = f32(1.0) + f32(2.0 ** -12)  # a^2 = 1 + 2^-11 + 2^-24, a midpoint of the fp32 grid near 1
    c[:250] = f32(2.0 ** -13)  # still a midpoint: ties to even
    c[250:375] = f32(2.0 ** -80)  # the fp64 sum rounds onto the midpoint, the exact one lies above it
    c[375:500] = f32(-(2.0 ** -80))
    got = KO.fma32(a, a, c)
    for x, y, g in zip(a.tolist(), c.tolist(), got.tolist()):
        exact = Fraction(x) * Fraction(x) + Fraction(y)
        lo = f32(float(exact))
        cands = {float(lo), float(np.nextafter(lo, f32(np.inf))), float(np.nextafter(lo, f32(-np.inf)))}
        best = min(cands, key=lambda v: (abs(Fraction(v) - exact), int(np.array(v, f32).view(np.int32)) & 1))
        assert g == best, (x, y, g, best)


@pytest.mark.parametrize("seed", range(4))
def test_restatement_equals_brute_force(seed):
    rng = np.random.default_rng(seed)
    n = [70, 150, 300, 200][seed]
    P = rng.uniform(-1, 1, (n, 3)).astype(f32)
    if seed == 1:
        P = np.round(P * 3).astype(f32)  # a lattice: massive ties
    if seed == 2:
        P[50:80] = P[:30]  # duplicates
        P[100:105] = [[np.nan, 0, 0], [np.inf, 1, 1], [0, -np.inf, 0], [np.nan] * 3, [1e30, 1e30, 1e30]]
    if seed == 3:
        P *= f32(1e-20)  # subnormal squares
        P[:3] += f32(3e18)  # squares beyond FLT_MAX
    want = KO.brute_knn3_mean_dist2(P)
    got = KO.knn3_mean_dist2(P)
    assert np.array_equal(got.view(np.int32), want.view(np.int32))


def test_small_clouds_and_non_finite_rows():
    P1 = np.array([[0.5, 0.25, -1.0]], f32)
    assert KO.knn3_mean_dist2(P1).tolist() == [math.inf]
    assert KO.knn3_mean_dist2(P1[:0]).shape == (0,)
    P2 = np.array([[0, 0, 0], [1, 0, 0]], f32)
    assert KO.knn3_mean_dist2(P2).tolist() == [math.inf, math.inf]
    P3 = np.array([[0, 0, 0], [1, 0, 0], [0, 2, 0]], f32)
    out = KO.knn3_mean_dist2(P3)
    FM = np.finfo(f32).max
    want0 = (f32(f32(1) + f32(4)) + FM) / f32(3)
    assert out[0] == want0 and np.isfinite(out).all() and abs(float(out[0]) - 1.13e38) < 0.01e38
    assert np.array_equal(out, KO.brute_knn3_mean_dist2(P3))
    # NaN and inf rows: +inf themselves, and invisible to every other point
    P = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1], [np.nan, 0, 0], [0, np.inf, 0], [0.1, 0, 0]], f32)
    out = KO.knn3_mean_dist2(P)
    ref = KO.knn3_mean_dist2(P[[0, 1, 2, 3, 6]])
    assert np.isinf(out[4]) and np.isinf(out[5]) and np.array_equal(out[[0, 1, 2, 3, 6]], ref)
    # a duplicate point contributes 0
    D = np.array([[0, 0, 0], [0, 0, 0], [3, 0, 0], [0, 4, 0]], f32)
    assert KO.knn3_mean_dist2(D)[0] == f32(f32(0 + 9) + 16) / f32(3)


def test_result_does_not_depend_on_row_order():
    rng = np.random.default_rng(7)
    P = rng.normal(size=(2000, 3)).astype(f32)
    P[:100] = np.round(P[:100])
    perm = rng.permutation(len(P))
    a, b = KO.knn3_mean_dist2(P), KO.knn3_mean_dist2(P[perm])
    assert np.array_equal(a[perm], b)


def _random_quat_tensor(n, g):
    """random_quat_tensor(N) (gauss_utils.hpp:32-46) statement by statement: u, v, w, then q1..q4 and the stack."""
    u, v, w = torch.rand(n, generator=g), torch.rand(n, generator=g), torch.rand(n, generator=g)
    two_pi = torch.tensor(2 * math.pi, dtype=torch.float32)  # ATen multiplies a float tensor by the double M_PI as a float
    q1 = torch.sqrt(torch.ones(()) - u) * torch.sin(two_pi * v)
    q2 = torch.sqrt(torch.ones(()) - u) * torch.cos(two_pi * v)
    q3 = torch.sqrt(u) * torch.sin(two_pi * w)
    q4 = torch.sqrt(u) * torch.cos(two_pi * w)
    return torch.stack([q1, q2, q3, q4], -1)


@pytest.mark.parametrize("n", [0, 1, 17, 5000])
def test_random_quat_matches_the_reference_statements(n):
    from gssdf_b200 import gs_init
    got = gs_init.random_quat(n, torch.Generator().manual_seed(3))
    want = _random_quat_tensor(n, torch.Generator().manual_seed(3))
    assert got.dtype == torch.float32 and tuple(got.shape) == (n, 4) and got.device.type == "cpu"
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))
    if n:
        assert torch.allclose(got.norm(dim=1), torch.ones(n), atol=1e-5)


@pytest.mark.parametrize("n", [0, 1, 2, 5, 999_999, 1_000_000, 1_999_999, 2_000_000, 2_000_001, 3_500_000, 16_777_217, 30_000_001])
def test_init_point_indices(n):
    from gssdf_b200 import gs_init
    r = gs_init.init_point_indices(n)
    step = max(int(f32(f32(n) / f32(1e6))), 1)  # int sample_step = N / 1e6f; max(step, 1)
    assert r == range(0, max(n - 1, 0), step)
    if n <= 2_000_001:  # slice(0, 0, -1, step) of a tensor with n rows
        assert torch.arange(n)[0:-1:step].tolist() == list(r)


def test_cabi_exports_and_rejects_without_launch():
    from gssdf_b200 import _lib
    L = _lib.lib()
    for sym in ("gssdf_knn3_mean_dist2", "gssdf_knn3_mean_dist2_workspace_bytes"):
        assert sym in _lib.FUNCS and hasattr(L, sym)
    assert L.gssdf_abi_revision() == 18
    assert L.gssdf_knn3_mean_dist2_workspace_bytes(1000) >= 40 * 1000
    assert L.gssdf_knn3_mean_dist2_workspace_bytes(-1) == 0 and L.gssdf_knn3_mean_dist2_workspace_bytes(2 ** 31) == 0
    assert L.gssdf_knn3_mean_dist2_workspace_bytes(2 ** 31 - 1) > 0 and L.gssdf_knn3_mean_dist2_workspace_bytes(0) > 0

    def call(**over):
        kw = dict(n=1000, points=0x1000, out=0x2000, workspace=0x3000, workspace_bytes=L.gssdf_knn3_mean_dist2_workspace_bytes(1000))
        kw.update(over)
        a = _lib.make_args("gssdf_knn3_mean_dist2_args", **kw)
        return L.gssdf_knn3_mean_dist2(C.byref(a), None), L.gssdf_last_error().decode()

    for over, word in ((dict(n=-1), "n must"), (dict(n=2 ** 31), "n must"), (dict(points=None), "required"), (dict(out=None), "required"),
                       (dict(workspace=None), "required"), (dict(workspace_bytes=L.gssdf_knn3_mean_dist2_workspace_bytes(1000) - 1), "workspace")):
        rc, msg = call(**over)
        assert rc == -1 and word in msg, (over, msg)
    assert L.gssdf_knn3_mean_dist2(None, None) == -1
    # n == 0 is a no-op that needs no pointers
    rc, _ = call(n=0, points=None, out=None, workspace=None, workspace_bytes=L.gssdf_knn3_mean_dist2_workspace_bytes(0))
    assert rc == 0


def test_dist_cuda2_argument_errors_without_a_gpu():
    from gssdf_b200 import gs_init
    with pytest.raises(ValueError, match="CUDA"):
        gs_init.dist_cuda2(torch.zeros(5, 3))
    with pytest.raises(ValueError, match=r"\[P,3\]"):
        gs_init.dist_cuda2(torch.zeros(5, 2))
    with pytest.raises(ValueError, match=r"\[P,3\]"):
        gs_init.dist_cuda2(torch.zeros(15))
    with pytest.raises(ValueError, match=r"\[n,3\]|CUDA"):
        gs_init.neural_gs_init_points(torch.zeros(5, 3), leaf_size=0.1, sh_degree=3, spatial_scale=1.0, inner_map_size=14.0,
                                      map_origin=(0, 0, 0))
