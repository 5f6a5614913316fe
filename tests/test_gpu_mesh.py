"""f-5 on the H100: gssdf_marching_cubes against its numpy restatement (bit-identical vertices, identical faces in the same order) and
against the reference's own kernels run live (oracle/_ref/cumcubes_ref.so), determinism, and the capacity / overflow contract."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import mesh_oracle as M

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def _edge_fields():
    rng = np.random.default_rng(3)
    out = {f"shape{s}": (rng.standard_normal(s).astype(np.float32), 0.0, [0.0, 0.0, 0.0], [1.0, 2.0, 3.0])
           for s in [(1, 1, 1), (1, 5, 6), (2, 2, 2), (2, 3, 1), (2, 7, 2), (3, 1, 4), (65, 3, 2)]}
    out["all_inside"] = (np.ones((6, 7, 8), np.float32), 0.0, [0.0] * 3, [1.0] * 3)
    out["all_outside"] = (-np.ones((6, 7, 8), np.float32), 0.0, [0.0] * 3, [1.0] * 3)
    out["equal_thresh"] = (rng.choice(np.float32([0.0, 1.0, -1.0]), (9, 9, 9)), 0.0, [0.0] * 3, [1.0] * 3)
    return out


@pytest.mark.parametrize("name", list(M.test_fields()) + list(_edge_fields()))
def test_marching_cubes_equals_oracle(name):
    from gssdf_b200 import mesh
    dev = _dev()
    g, t, lo, hi = {**M.test_fields(), **_edge_fields()}[name]
    v, f = mesh.marching_cubes(torch.from_numpy(g).to(dev), t, lo, hi)
    rv, rf, _ = M.marching_cubes(g, t, lo, hi)
    assert np.array_equal(v.cpu().numpy().view(np.uint32), rv.view(np.uint32))
    assert np.array_equal(f.cpu().numpy(), rf)


@pytest.mark.parametrize("name", list(M.test_fields()))
def test_marching_cubes_vs_reference_kernels_live(name):
    """The reference's mc::marching_cubes on the same field, compared by table-independent invariants (its case table is not ours).
    Agreement of the per-cell vector areas also shows that the reference orients its triangles like we do: normal toward increasing
    value."""
    from gssdf_b200 import mesh
    dev = _dev()
    if not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "cumcubes_ref.so")):
        pytest.skip("oracle/_ref/cumcubes_ref.so not built (oracle/build_ref_mc.py)")
    import importlib.util
    spec = importlib.util.spec_from_file_location("gen_golden_mc", os.path.join(ROOT, "oracle", "gen_golden_mc.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    g, t, lo, hi = M.test_fields()[name]
    ref_v, ref_f = gen.run(gen.load_ref(), g, t, lo, hi)
    r = M.compare_with_reference(g, t, lo, hi, ref_v, ref_f)
    print(name, r)
    v, f = mesh.marching_cubes(torch.from_numpy(g).to(dev), t, lo, hi)
    rv, rf, _ = M.marching_cubes(g, t, lo, hi)
    assert np.array_equal(v.cpu().numpy().view(np.uint32), rv.view(np.uint32)) and np.array_equal(f.cpu().numpy(), rf)


def test_marching_cubes_is_deterministic_on_a_large_field():
    from gssdf_b200 import mesh
    dev = _dev()
    gen = torch.Generator(device=dev).manual_seed(0)
    g = torch.randn(160, 150, 140, device=dev, generator=gen)
    v1, f1 = mesh.marching_cubes(g, 0.1, [0, 0, 0], [1, 1, 1])
    v2, f2 = mesh.marching_cubes(g, 0.1, [0, 0, 0], [1, 1, 1])
    assert len(f1) > 1_000_000
    assert torch.equal(v1, v2) and torch.equal(f1, f2)
    gc = g.cpu().numpy()
    rv, rf, _ = M.marching_cubes(gc, 0.1, [0, 0, 0], [1, 1, 1])
    assert np.array_equal(v1.cpu().numpy().view(np.uint32), rv.view(np.uint32)) and np.array_equal(f1.cpu().numpy(), rf)


def test_capacity_overflow_writes_nothing_past_the_capacity():
    """C ABI: with too-small capacities the true counts and the overflow bits are reported, the rows below the capacities hold the start of
    the full output, and a guard region after each buffer is untouched. mesh.marching_cubes started too small retries once with the
    exact counts and returns the full mesh."""
    from gssdf_b200 import cabi, mesh
    from gssdf_b200._lib import check, lib, make_args
    dev = _dev()
    g, t, lo, hi = M.test_fields()["random"]
    rv, rf, _ = M.marching_cubes(g, t, lo, hi)
    vcap, fcap, guard = 1000, 700, 64
    gt = torch.from_numpy(g).to(dev)
    vbuf = torch.full((vcap + guard, 3), 12345.0, device=dev)
    fbuf = torch.full((fcap + guard, 3), -7, dtype=torch.int32, device=dev)
    counts = torch.full((4,), -1, dtype=torch.int32, device=dev)
    nx, ny, nz = g.shape
    ws = torch.empty(lib().gssdf_marching_cubes_workspace_bytes(nx, ny, nz), dtype=torch.uint8, device=dev)
    a = make_args("gssdf_marching_cubes_args", nx=nx, ny=ny, nz=nz, grid=gt, thresh=t, lower=lo, upper=hi, vertex_cap=vcap, face_cap=fcap,
                  vertices=vbuf, faces=fbuf, counts=counts, workspace=ws, workspace_bytes=ws.numel())
    check(lib().gssdf_marching_cubes(C.byref(a), cabi._stream()))
    assert counts.tolist() == [len(rv), len(rf), 3, 0]
    assert np.array_equal(vbuf[:vcap].cpu().numpy(), rv[:vcap]) and np.array_equal(fbuf[:fcap].cpu().numpy(), rf[:fcap])
    assert bool((vbuf[vcap:] == 12345.0).all()) and bool((fbuf[fcap:] == -7).all())
    a.workspace_bytes = ws.numel() - 1
    with pytest.raises(Exception, match="workspace"):
        check(lib().gssdf_marching_cubes(C.byref(a), cabi._stream()))
    v, f = mesh.marching_cubes(gt, t, lo, hi, vertex_cap=10, face_cap=10)
    assert np.array_equal(v.cpu().numpy(), rv) and np.array_equal(f.cpu().numpy(), rf)


@pytest.mark.parametrize("name", ["random", "sphere", "ambiguous"])
def test_cumcubes_shim_twin_equals_the_operator(name):
    """mc::marching_cubes of the libtorch twin (what LocalMap::meshing_ links against) returns the operator's mesh; the random field
    outgrows the twin's first capacity guess, so its retry with the exact counts is exercised too."""
    import gssdf_shim as shim

    from gssdf_b200 import mesh
    dev = _dev()
    g, t, lo, hi = M.test_fields()[name]
    gt = torch.from_numpy(g).to(dev)
    v, f = shim.mc_marching_cubes(gt, t, lo, hi)
    v2, f2 = mesh.marching_cubes(gt, t, lo, hi)
    assert v.dtype == torch.float32 and f.dtype == torch.int32 and v.is_cuda and f.is_cuda
    assert torch.equal(v, v2) and torch.equal(f, f2)
    if name == "random":
        assert len(v) > max(g.size // 16, 1024)
