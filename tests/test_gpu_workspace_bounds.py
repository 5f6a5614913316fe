"""Workspace bounds of every operator that takes a caller-owned workspace: each call accepts a workspace of exactly the size its
gssdf_*_workspace_bytes advertises, rejects one byte less with the documented code and a message about the workspace, and writes
nothing past the advertised size. The operators run through the package's own wrappers on a stand-in for cabi.Workspace whose buffers
are exact-size views of a larger allocation with a sentinel tail."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

EINVAL, ENOMEM = -1, -4
# entry point -> error code for a workspace one byte short (include/gssdf_b200.h)
SHORT_CODE = {
    "gssdf_project2dgs_fwd": ENOMEM, "gssdf_tile_encode": ENOMEM, "gssdf_raster2dgs_fwd": ENOMEM, "gssdf_raster2dgs_bwd": ENOMEM,
    "gssdf_dssim_loss": ENOMEM, "gssdf_octree_raytrace": ENOMEM, "gssdf_sdf_sample_rays": ENOMEM, "gssdf_sdf_gate_compact": ENOMEM,
    "gssdf_marching_cubes": ENOMEM, "gssdf_sdf_mesh": ENOMEM, "gssdf_octree_build": ENOMEM, "gssdf_sdf_init_gs": EINVAL,
    "gssdf_mesh_cull_faces": EINVAL, "gssdf_mesh_sample_uniform": EINVAL, "gssdf_voxel_downsample": EINVAL, "gssdf_nn_truncated": EINVAL,
}
SENTINEL, PAD = 0xA5, 4096


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


class GuardedWorkspace:
    """cabi.Workspace with exact sizes: get(n) returns (and .buf is) the first n bytes of a larger buffer whose tail holds SENTINEL.
    The tail is checked before it is re-laid and by verify()."""
    instances = []

    def __init__(self, device):
        self.device, self.buf, self._base, self._n = device, None, None, 0
        GuardedWorkspace.instances.append(self)

    def get(self, nbytes):
        self.verify()
        n = int(nbytes)
        if self._base is None or self._base.numel() < n + PAD:
            self._base = torch.empty(n + PAD, dtype=torch.uint8, device=self.device)
        self._base[n:].fill_(SENTINEL)
        self._n, self.buf = n, self._base[:n]
        return self.buf

    def verify(self):
        if self._base is not None:
            tail = self._base[self._n:]
            assert bool((tail == SENTINEL).all()), f"an operator wrote past the advertised {self._n} workspace bytes"


@pytest.fixture
def guarded(monkeypatch):
    """Patches cabi.Workspace with GuardedWorkspace and wraps the entry points: returns (calls made, set_short(name)). With
    set_short(name), every call of that entry point is told its workspace is one byte smaller than the advertised size."""
    from gssdf_b200 import _lib, cabi
    _dev()
    GuardedWorkspace.instances = []
    monkeypatch.setattr(cabi, "Workspace", GuardedWorkspace)
    L, calls, short = _lib.lib(), [], [None]
    for name in SHORT_CODE:
        def call(aref, stream, _fn=getattr(L, name), _name=name):
            calls.append(_name)
            if _name == short[0]:
                aref._obj.workspace_bytes -= 1
            return _fn(aref, stream)
        monkeypatch.setattr(L, name, call)
    yield calls, lambda name: short.__setitem__(0, name)
    torch.cuda.synchronize()
    for ws in GuardedWorkspace.instances:
        ws.verify()


# ---- one representative workload per group of operators; each returns nothing and runs on cabi.Workspace ----
def render_step(dev):
    from gssdf_b200 import render
    from gssdf_b200 import scene as S
    N, W, H, deg = 4000, 160, 96, 3
    sc = S.box_scene(N, deg, seed=0, scale_mult=6.0)
    V, K = S.cameras([0], W, H)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    R = render.SplatRenderer(N, (deg + 1) ** 2, 1, W, H, dev, isect_cap=300000, sh_degree=deg)
    sc = {k: t(v) for k, v in sc.items()}
    splats = (sc["means"], sc["quats"], sc["scales"], sc["opacities"], sc["sh"], t(V), t(K))
    rn = t(S.randns(N))
    R.forward(*splats, rn, raw=sc.get("raw"))
    R.backward(*splats, torch.rand(1, H, W, 4, device=dev), rn, raw=sc.get("raw"), w_dssim=0.2)  # w_dssim > 0 runs gssdf_dssim_loss


def gate_compact(dev):
    from gssdf_b200 import cabi
    n = 5000
    g = torch.Generator(device=dev).manual_seed(0)
    x, vis = torch.rand(n, 3, device=dev, generator=g), torch.rand(n, device=dev, generator=g)
    idx, xo, ng = torch.empty(n, dtype=torch.int32, device=dev), torch.empty(n, 3, device=dev), torch.zeros(1, dtype=torch.int32, device=dev)
    cabi.sdf_gate_compact(n, x, idx, xo, ng, cabi.Workspace(dev), visibilities=vis, visible_thr=0.5)


def _room_points(rng, n):
    """points on the walls of a 6 x 4 x 3 m box"""
    p = rng.uniform(-1, 1, (n, 3)).astype(np.float32)
    axis = rng.integers(0, 3, n)
    p[np.arange(n), axis] = np.sign(p[np.arange(n), axis])
    return p * np.float32([3, 2, 1.5])


def raytrace_and_sample(dev):
    from gssdf_b200 import octree as OT
    rng = np.random.default_rng(0)
    level, map_size, n_rays = 7, 14.0, 3000
    surf = _room_points(rng, 50000)
    tree = OT.OctreeAS.from_quantized_points(OT.quantize_points(torch.from_numpy(surf * np.float32(2 / map_size)).to(dev), level).cpu(),
                                             level, dev, map_size=map_size)
    origin = (rng.uniform(-0.5, 0.5, (n_rays, 3)) * [3, 2, 1.5]).astype(np.float32)
    end = surf[rng.integers(0, len(surf), n_rays)]
    depth = np.linalg.norm(end - origin, axis=1).astype(np.float32)
    direction = ((end - origin) / depth[:, None]).astype(np.float32)
    t = lambda a: torch.from_numpy(a).to(dev)
    tree.raytrace(t(origin), t(direction))
    S = OT.RaySampler(tree, n_rays, dev, 1, 4, 3, 0.1, 0.3, (-7,) * 3, (7,) * 3)
    S.draw()
    S.sample(t(origin), t(direction), t(depth), t(end))


def octree_build(dev):
    """both calls of gssdf_octree_build (update_octree_as allocates its own workspace)"""
    from gssdf_b200 import _lib, cabi
    level, map_size = 7, 14.0
    x = torch.from_numpy(_room_points(np.random.default_rng(1), 20000)).to(dev)
    ws = cabi.Workspace(dev).get(_lib.lib().gssdf_octree_build_workspace_bytes(C.c_int64(x.shape[0]), level))
    counts = torch.zeros(level + 2, dtype=torch.int64, device=dev)
    a = _lib.make_args("gssdf_octree_build_device_args", n=x.shape[0], xyz=x, origin=[0.0, 0.0, 0.0], inv_size=1.0 / map_size, level=level,
                       dilate=1, counts=counts, workspace=ws, workspace_bytes=ws.numel())
    _lib.check(_lib.lib().gssdf_octree_build(C.byref(a), cabi._stream()))
    c = counts.tolist()
    npnt = sum(c[:level + 1])
    nn = npnt - c[level]
    outs = (torch.empty(max(nn, 1), dtype=torch.uint8, device=dev), torch.empty(nn + 1, dtype=torch.int32, device=dev),
            torch.empty(max(npnt, 1), 3, dtype=torch.int16, device=dev), torch.empty(2, level + 2, dtype=torch.int32, device=dev))
    a.node_cap, a.point_cap = nn, npnt
    a.octree, a.exsum, a.points, a.pyramid = (o.data_ptr() for o in outs)
    _lib.check(_lib.lib().gssdf_octree_build(C.byref(a), cabi._stream()))


def marching_cubes(dev):
    from gssdf_b200 import mesh
    n = (40, 41, 42)
    axes = [torch.linspace(-1, 1, k, device=dev) for k in n]
    X, Y, Z = torch.meshgrid(*axes, indexing="ij")
    mesh.marching_cubes((X * X + Y * Y + Z * Z).sqrt().sub(0.7).contiguous(), 0.0, [-1.0] * 3, [1.0] * 3)


def _random_net(dev, **kw):
    from gssdf_b200 import sdf as SD
    net = SD.SdfNet(dev, seed=1337, **kw)
    g = torch.Generator(device="cpu").manual_seed(0)
    with torch.no_grad():
        net.params_.copy_((torch.rand(net.params_.numel(), generator=g) - 0.5).to(dev))
    return net


def sdf_mesh(dev):
    from gssdf_b200 import mesh
    from gssdf_b200 import octree as OT
    level, leaf = 6, 0.1
    map_size = float(np.float32(2 ** level) * np.float32(leaf))
    rng = np.random.default_rng(2)
    shell = rng.normal(size=(20000, 3)).astype(np.float32)
    shell = shell / np.linalg.norm(shell, axis=1, keepdims=True) * np.float32(1.5)
    tree = OT.OctreeAS.from_quantized_points(OT.quantize_points(torch.from_numpy(shell * np.float32(2 / map_size)).to(dev), level).cpu(),
                                             level, dev, map_size=map_size)
    net = _random_net(dev, map_size=map_size)
    mesh.meshing(tree, net, (-2.95,) * 3, (2.95,) * 3, 0.05, color_mode=2)


def sdf_init_gs(dev):
    from gssdf_b200 import gs_init
    net = _random_net(dev, origin=(0.3, -0.2, 0.1), map_size=14.0, bce_isigma=10.0)
    x = ((torch.rand(5000, 3, generator=torch.Generator(device="cpu").manual_seed(3)) * 2 - 1) * 3.0).to(dev).contiguous()
    gs_init.sdf_init_gs(gs_init._net_struct(net), x, 0.01, 10.0, torch.empty(x.shape[0], 4, device=dev))


def mesh_cull(dev):
    from gssdf_b200 import cabi, mesh
    g = torch.Generator(device=dev).manual_seed(4)
    V, M = 3000, 7000
    faces = torch.randint(0, V, (M, 3), device=dev, generator=g, dtype=torch.int32)
    seen = (torch.rand(V, device=dev, generator=g) < 0.3).to(torch.uint8)
    out, counts = torch.empty(M, 3, dtype=torch.int32, device=dev), torch.zeros(2, dtype=torch.int32, device=dev)
    mesh.cull_faces(faces, V, seen, out, counts, cabi.Workspace(dev))


def eval_mesh(dev):
    from gssdf_b200 import mesh
    g = torch.Generator(device=dev).manual_seed(5)
    v = torch.rand(2000, 3, device=dev, generator=g)
    f = torch.randint(0, 2000, (4000, 3), device=dev, generator=g, dtype=torch.int32)
    mesh.eval_mesh(v, f, torch.rand(30000, 3, device=dev, generator=g), mesh_sample_point=200_000)


WORKLOADS = {
    render_step: ["gssdf_project2dgs_fwd", "gssdf_tile_encode", "gssdf_raster2dgs_fwd", "gssdf_dssim_loss", "gssdf_raster2dgs_bwd"],
    gate_compact: ["gssdf_sdf_gate_compact"],
    raytrace_and_sample: ["gssdf_octree_raytrace", "gssdf_sdf_sample_rays"],
    octree_build: ["gssdf_octree_build"],
    marching_cubes: ["gssdf_marching_cubes"],
    sdf_mesh: ["gssdf_sdf_mesh"],
    sdf_init_gs: ["gssdf_sdf_init_gs"],
    mesh_cull: ["gssdf_mesh_cull_faces"],
    eval_mesh: ["gssdf_mesh_sample_uniform", "gssdf_voxel_downsample", "gssdf_nn_truncated"],
}


def test_every_workspace_operator_is_covered():
    assert sorted(n for names in WORKLOADS.values() for n in names) == sorted(SHORT_CODE)


@pytest.mark.parametrize("run", list(WORKLOADS), ids=lambda f: f.__name__)
def test_exact_workspace_is_accepted_and_never_overrun(run, guarded):
    calls, _ = guarded
    run(_dev())
    assert set(WORKLOADS[run]) <= set(calls), calls


@pytest.mark.parametrize("run,name", [(f, n) for f, names in WORKLOADS.items() for n in names], ids=lambda v: getattr(v, "__name__", v))
def test_one_byte_short_is_rejected(run, name, guarded):
    from gssdf_b200 import _lib
    calls, set_short = guarded
    set_short(name)
    with pytest.raises((ValueError, _lib.GssdfError), match="workspace") as e:
        run(_dev())
    assert calls[-1] == name
    assert (e.value.code if isinstance(e.value, _lib.GssdfError) else EINVAL) == SHORT_CODE[name]
