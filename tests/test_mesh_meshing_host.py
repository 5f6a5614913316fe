"""f-5 second stage on the CPU: the numpy restatement of the global-lattice meshing (tests/meshing_oracle.py) against a brute-force
boundary filter, against the literal restatement of the reference's slab walk (one slab: identical; many slabs: the same surface up to
the slab origins' rounding), the lattice rule against torch.arange,, the C ABI's argument checks (no launch) and the libtorch meshing entry point in the shim."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

import meshing_oracle as MO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32
LEVEL, LEAF = 5, 0.1
MAP = float(f32(f32(2 ** LEVEL) * f32(LEAF)))


def _scene(origin=(0.0, 0.0, 0.0)):
    tree, _ = MO.shell_tree(MO.sphere_points(np.asarray(origin) + [0.05, -0.1, 0.08], 0.9), LEVEL, MAP, origin)
    return MO.Occupancy(tree, origin, MAP)


def _fields(origin):
    c = np.asarray(origin, np.float64) + [0.05, -0.1, 0.08]
    rng = np.random.default_rng(1)
    k = rng.normal(size=(4, 3)) * 3
    return {
        "sphere": lambda p: (0.9 - np.linalg.norm(p - c, axis=1)).astype(f32),
        "box": lambda p: (0.7 - np.abs(p - c).max(1)).astype(f32),
        "random": lambda p: (np.sin(p @ k.T).sum(1) * 0.3 + 0.05).astype(f32),
    }


MARGIN = ((-1.55,) * 3, (1.55,) * 3)


@pytest.mark.parametrize("field", ["sphere", "box", "random"])
def test_meshing_filter_equals_brute_force(oracle, field):
    occ = _scene()
    lower, n = MO.lattice(*MARGIN, (0.0, 0.0, 0.0), 0.05)
    r = MO.meshing(lower, n, 0.05, occ, _fields((0.0, 0.0, 0.0))[field])
    v, f, keep = r["raw_vertices"], r["raw_faces"], r["face_keep"]
    assert len(f) > 100 and 0 < keep.sum() < len(f)
    vpass = np.zeros(len(v), bool)
    inv = f32(f32(1.0) / f32(0.05))  # ATen on CUDA: tensor / CPU scalar = tensor * fp32 reciprocal
    for i in range(len(v)):  # per vertex: floor(v / res) -> int16, its 27 neighbours * res, all occupied
        q = np.floor(v[i] * inv).astype(np.int16)
        pts = [np.array([q[0] + a, q[1] + b, q[2] + c], np.int16).astype(f32) * f32(0.05) for a in (-1, 0, 1) for b in (-1, 0, 1) for c in (-1, 0, 1)]
        vpass[i] = bool(occ(np.stack(pts)).all())
    want = np.array([vpass[a] and vpass[b] and vpass[c] for a, b, c in f])
    assert np.array_equal(keep, want)
    fk = f[want]
    used = np.unique(fk)
    assert np.array_equal(r["vertices"], v[used]) and np.array_equal(used[r["faces"]], fk)


@pytest.mark.parametrize("origin", [(0.0, 0.0, 0.0), (0.3, -0.15, 0.2)])
def test_one_slab_equals_the_reference_walk(oracle, origin):
    occ = _scene(origin)
    fn = _fields(origin)["random"]
    res = 0.05
    lower, n = MO.lattice(*MARGIN, origin, res)
    ours = MO.meshing(lower, n, res, occ, fn)
    rv, rf = MO.meshing_reference_slabs(*MARGIN, origin, res, occ, fn)
    assert len(ours["faces"]) > 100
    tri = lambda v, f: v[f].view(np.uint32).reshape(len(f), -1)
    assert np.array_equal(tri(ours["vertices"], ours["faces"]), tri(rv, rf))


def test_many_slabs_give_the_same_surface(oracle):
    from scipy.spatial import cKDTree
    occ = _scene()
    fn = _fields((0.0, 0.0, 0.0))["sphere"]
    res = 0.05
    lower, n = MO.lattice(*MARGIN, (0.0, 0.0, 0.0), res)
    ours = MO.meshing(lower, n, res, occ, fn)
    rv, rf = MO.meshing_reference_slabs(*MARGIN, (0.0, 0.0, 0.0), res, occ, fn, batch_pt_num=4000)
    # a slab whose arange length ATen's ceil rounds up reaches one lattice plane into the next slab: the cells between the two planes
    # are meshed by both slabs, so those triangles appear twice in the reference's output; drop the second copies
    cen = rv[rf].astype(np.float64).mean(1)
    dup = np.zeros(len(rf), bool)
    for i, j in cKDTree(cen).query_pairs(1e-4 * res):
        dup[max(i, j)] = True
    assert dup.any()
    rf = rf[~dup]
    a0, a1 = MO.area(ours["vertices"], ours["faces"]), MO.area(rv, rf)
    assert abs(a0 - a1) <= 1e-5 * a0
    used = np.unique(rf)
    d01 = cKDTree(rv[used]).query(ours["vertices"])[0].max()
    d10 = cKDTree(ours["vertices"]).query(rv[used])[0].max()
    assert max(d01, d10) <= 1e-4 * res, (d01, d10)
    assert len(used) > len(ours["vertices"])  # the seams repeat vertices


@pytest.mark.parametrize("box,res", [((-1.55, 1.55), 0.05), ((-6.975, 6.975), 0.01), ((-2.95, 3.1), 0.037), ((0.1, 0.71), 0.0123),
                                     ((-7.0 + 0.025, 7.0 - 0.025), 0.04), ((-3.33, 2.2), 0.025)])
@pytest.mark.parametrize("center", [0.0, 0.35, -1.7])
def test_lattice_rule_matches_torch_arange(box, res, center):
    from gssdf_b200 import mesh
    lo, hi = box
    lower, n = mesh.lattice((lo,) * 3, (hi,) * 3, (center,) * 3, res)
    start = f32(f32(lo) + f32(center))
    end = f32(f32(f32(hi) + f32(center)) + f32(res))
    t = torch.arange(float(start), float(end), float(f32(res)))  # reference: torch::arange(float, float, float)
    assert n == [t.numel()] * 3 and lower == [float(start)] * 3
    assert (MO.lattice((lo,) * 3, (hi,) * 3, (center,) * 3, res)[1]) == n


def _args(**kw):
    from gssdf_b200 import _lib
    a = _lib.make_args("gssdf_sdf_mesh_args", **kw)
    return a


def _call(a):
    from gssdf_b200 import _lib
    rc = _lib.lib().gssdf_sdf_mesh(C.byref(a), None)
    return rc, _lib.lib().gssdf_last_error().decode()


def _valid_args(**over):
    """An argument set that passes every check up to the launch; pointers are dummies (never dereferenced on a rejection)."""
    kw = dict(leaves=0x1000, n_leaves=10, lower=[-7.0, -7.0, -7.0], n=[100, 100, 100], res=0.05, color_mode=0, vertex_cap=10, face_cap=10,
              vertices=0x2000, faces=0x3000, colors=0x4000, counts=0x5000, workspace=None, workspace_bytes=0)
    kw.update(over)
    a = _args(**kw)
    a.tree.level, a.tree.n_nodes, a.tree.octree, a.tree.exsum, a.tree.inv_size, a.tree.size = 9, 10, 0x6000, 0x7000, 1 / 25.6, 25.6
    a.net.table_half, a.net.mlp = 0x8000, 0x9000
    return a


def test_cabi_rejects_without_launch():
    from gssdf_b200 import _lib
    L = _lib.lib()
    rc, msg = _call(_valid_args())
    assert rc == -4 and "workspace" in msg  # missing workspace
    assert L.gssdf_sdf_mesh_workspace_bytes(C.byref(_valid_args())) > 0
    for res in (0.0, -0.05, float("nan")):
        rc, msg = _call(_valid_args(res=res))
        assert rc == -1 and "res" in msg
        assert L.gssdf_sdf_mesh_workspace_bytes(C.byref(_valid_args(res=res))) == 0
    # int16: |coordinate / res| + 1 must stay below 32768 (the filter's cast of floor(v / res))
    rc, msg = _call(_valid_args(lower=[-7.0, -7.0, -7.0], n=[100, 100, 100], res=0.0002))
    assert rc == -1 and "int16" in msg
    rc, msg = _call(_valid_args(lower=[-7.0, 400.0, -7.0], res=0.01))
    assert rc == -1 and "int16" in msg
    rc, _ = _call(_valid_args(color_mode=3))
    assert rc == -1


def test_shim_header_compiles_into_the_shim():
    """shim/include/gssdf_mesh.hpp is compiled into gssdf_shim.so (build() builds it): gssdf::meshing_ is defined there with the
    declared signature."""
    import shutil
    so = os.path.join(ROOT, "gs-sdf_b200", "gssdf_shim.so")
    assert os.path.exists(so), "gssdf_shim.so is built by build()"
    nm = shutil.which("nm")
    if nm is None:
        pytest.skip("needs binutils' nm")
    out = subprocess.run([nm, "-DC", "--defined-only", so], capture_output=True, text=True, check=True).stdout
    sig = ("gssdf::meshing_(at::Tensor const&, at::Tensor const&, at::Tensor const&, at::Tensor const&, int, TCNNEncoding const&, "
           "torch::nn::Sequential&, at::Tensor const&, at::Tensor const&, at::Tensor const&, float, float, int, bool)")
    assert sig in out
    src = open(os.path.join(ROOT, "gs-sdf_b200", "shim", "gssdf_mesh.cpp")).read()
    assert '#include "gssdf_mesh.hpp"' in src


def test_arange_emulation_rounds_once():
    """arange_cuda rounds start + i * step once: against exact rational arithmetic, including values built to land on float32 ties."""
    from fractions import Fraction
    rng = np.random.default_rng(5)
    cases = [(-6.975, 0.01), (-2.95, 0.037), (1e-3, 0.0123), (-1e4, 3.3e-3), (float(f32(2.0 ** 20)), float(f32(2.0 ** -30) * 3))]
    cases += [(float(f32(rng.uniform(-50, 50))), float(f32(10 ** rng.uniform(-4, 0)))) for _ in range(20)]
    for start, step in cases:
        got = MO.arange_cuda(start, step, 3000)
        for i in range(0, 3000, 7):
            x = Fraction(float(f32(start))) + i * Fraction(float(f32(step)))
            c = f32(float(x))  # float64 nearest, then float32: compare with the two float32 neighbours exactly
            cands = [c, np.nextafter(c, f32(np.inf)), np.nextafter(c, f32(-np.inf))]
            best = min(cands, key=lambda y: (abs(Fraction(float(y)) - x), int(np.asarray(y).view(np.uint32)) & 1))
            assert got[i] == best, (start, step, i)
