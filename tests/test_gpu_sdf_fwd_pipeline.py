"""The tensor-core SDF forward (gssdf_sdf_fwd, mlp_mode 1) computes every row on its own: a row's sdf / y1 / feat must not depend on
which 128-row tile, which CTA or which feature buffer of the encode pipeline it went through. The same points are evaluated grouped
differently -- permuted, at another capacity stride with a device live count, with skip_base_variant, in batches of 1, 127, 128, 129
tiles and in one of far more tiles than CTAs -- and every row must come out bit-identical (torch.equal)."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

M = 40037           # points: 7 variants -> 2225 tiles of 18 points (more than 2 per CTA on any current GPU)
DELTA = 0.01


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def setup():
    from gssdf_b200 import cabi
    dev = _dev()
    rng = np.random.default_rng(2024)
    n_params = cabi.sdf_table_params(cabi.sdf_net(torch.zeros(1, device=dev), torch.zeros(1, device=dev)))
    table = torch.from_numpy(rng.uniform(-0.5, 0.5, n_params).astype(np.float32)).to(dev)
    dims, ps = [32, 64, 64, 64, 64, 2], []
    for k, o in zip(dims[:-1], dims[1:]):
        b = 1 / np.sqrt(k)
        ps += [rng.uniform(-b, b, o * k), rng.uniform(-b, b, o)]
    mlp = torch.from_numpy(np.concatenate(ps).astype(np.float32)).to(dev)
    half = torch.empty(n_params, dtype=torch.float16, device=dev)
    cabi.sdf_table_to_half(table, half)
    probe = cabi.sdf_net(half, mlp)
    packed = torch.empty(cabi.sdf_mlp_packed_bytes(probe), dtype=torch.uint8, device=dev)
    cabi.sdf_mlp_pack(probe, packed)
    net = cabi.sdf_net(half, mlp, mlp_mode=1, mlp_packed=packed)
    x = torch.from_numpy(rng.uniform(0.02, 0.98, (M, 3)).astype(np.float32)).to(dev)
    ref = _run(net, x, 7)
    return dict(net=net, keep=(half, mlp, packed), x=x, ref=ref, dev=dev)


def _run(net, x, nv, n_live=None, skip=False):
    """sdf, y1, feat of every evaluation, [nv][n] rows; rows the launch does not write stay NaN"""
    from gssdf_b200 import cabi
    n = x.shape[0]
    out = [torch.full((nv * n,), float("nan"), device=x.device), torch.full((nv * n,), float("nan"), device=x.device),
           torch.full((nv * n, 32), float("nan"), device=x.device)]
    nl = torch.tensor([n_live], dtype=torch.int32, device=x.device) if n_live is not None else None
    cabi.sdf_fwd(net, x, out[0], out[1], out[2], n_variants=nv, delta=DELTA, n_live=nl, skip_base_variant=skip)
    torch.cuda.synchronize()
    return [o.view(nv, n, *o.shape[1:]) for o in out]


def _same(got, want):
    for g, w in zip(got, want):
        assert torch.equal(g, w), f"{int((g != w).sum())} of {g.numel()} values differ"


def test_permuted_rows(setup):
    perm = torch.from_numpy(np.random.default_rng(1).permutation(M)).to(setup["dev"])
    got = _run(setup["net"], setup["x"][perm].contiguous(), 7)
    _same(got, [r[:, perm] for r in setup["ref"]])


@pytest.mark.parametrize("cap", [M + 1, M + 5000, 3 * M + 77])
@pytest.mark.parametrize("skip", [False, True])
def test_capacity_stride_and_live_count(setup, cap, skip):
    """the points as the first M rows of a larger buffer (another stride n, device n_live = M); the rows beyond stay untouched"""
    x = torch.rand(cap, 3, device=setup["dev"], generator=torch.Generator(setup["dev"]).manual_seed(cap)) * 0.96 + 0.02
    x[:M] = setup["x"]
    got = _run(setup["net"], x, 7, n_live=M, skip=skip)
    v0 = 1 if skip else 0  # skip_base_variant: variant 0 is not part of the result
    _same([g[v0:, :M] for g in got], [r[v0:] for r in setup["ref"]])
    assert all(bool(torch.isnan(g[:, M:]).all()) for g in got)


def test_live_count_inside_a_tile(setup):
    """n_live that ends mid-tile, and a live count below the stride"""
    n_live = M - 1000 - 45
    got = _run(setup["net"], setup["x"], 7, n_live=n_live)
    _same([g[:, :n_live] for g in got], [r[:, :n_live] for r in setup["ref"]])
    assert all(bool(torch.isnan(g[:, n_live:]).all()) for g in got)


@pytest.mark.parametrize("tiles", [1, 127, 128, 129])
def test_batches_of_whole_tiles(setup, tiles):
    n = 128 * tiles
    got = _run(setup["net"], setup["x"][:n].contiguous(), 1)
    _same(got, [r[:1, :n] for r in setup["ref"]])


@pytest.mark.parametrize("n", [1, 127, 129, 1000])
def test_partial_last_tile(setup, n):
    """n not a multiple of the points per tile (128, or 18 with 7 variants): a partly filled last tile"""
    got = _run(setup["net"], setup["x"][:n].contiguous(), 7)
    _same(got, [r[:, :n] for r in setup["ref"]])
