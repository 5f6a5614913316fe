"""f-12 without a GPU: the row rule of sdf_train_callback's outlier branch (neural_mapping.cpp:559-592) against a literal torch CPU replay of
the reference's chunk loop, sdf.remove_outliers's plumbing on a CPU pack (the operator replaced by its header contract on the host), and
sdf.outlier_threshold bit for bit against the reference's expression compiled with g++."""
import struct
import subprocess

import numpy as np
import pytest
import torch

from gssdf_b200 import cabi
from gssdf_b200 import sdf as SD

f32 = np.float32
B = 7  # a small k_vis_batch_pt_num: the rule does not depend on it


def fake_sdf(xyz):
    """A row-independent stand-in for LocalMap::get_sdf(x)[0]: [m,1]."""
    return (xyz[:, :1] - 0.5).contiguous()


def replay(pack, thr, b):
    """sdf_train_callback's outlier branch, statement by statement, on the CPU with fake_sdf."""
    train_pcl = pack["xyz"].view(-1, 3)
    point_num = train_pcl.shape[0]
    inlier_idx_vec = []
    for i in range(0, point_num, b):
        end = min(i + b, point_num - 1)
        xyz_pred_sdf = fake_sdf(train_pcl.index_select(0, torch.arange(i, end)))
        inlier_idx = (xyz_pred_sdf.abs() < thr).squeeze().nonzero().squeeze().cpu()
        inlier_idx_vec.append(inlier_idx + i)
    inlier_idx = torch.cat(inlier_idx_vec, 0)
    return {k: v.index_select(0, inlier_idx) for k, v in pack.items()}


def evaluated_rows(N, b):
    """The rows the chunk loop hands to get_sdf."""
    rows = []
    for i in range(0, N, b):
        rows += list(range(i, min(i + b, N - 1)))
    return rows


def rule(xyz, thr, b=B):
    """The twin's rule: {r < outlier_rows(N, B) : |sdf_r| < thr}, ascending."""
    n = SD.outlier_rows(xyz.shape[0], b)
    s = fake_sdf(xyz[:n])[:, 0]
    return torch.nonzero(s.abs() < torch.tensor(thr, dtype=torch.float32)).view(-1)


def make_pack(N, seed, keep_pattern=None):
    g = torch.Generator().manual_seed(seed)
    xyz = torch.rand(N, 3, generator=g)
    if keep_pattern is not None:  # sdf 0 (kept) or 1 (dropped at every threshold used here) row by row
        xyz[:, 0] = torch.where(keep_pattern, torch.tensor(0.5), torch.tensor(1.5))
    return {"origin": torch.rand(N, 3, generator=g), "direction": torch.rand(N, 3, generator=g), "depth": torch.rand(N, 1, generator=g),
            "xyz": xyz}


class _FakeNet:
    """What remove_outliers reads of an SdfNet: the device and the C struct (unused by the fake operator)."""
    params_ = torch.zeros(1)
    decoder_ = torch.zeros(1)

    def _net(self, table, mlp):
        return None


@pytest.fixture
def host_operator(monkeypatch):
    """cabi.sdf_outlier_filter replaced by its header contract evaluated with fake_sdf (CPU index path only)."""
    calls = []

    def op(net, xyz, threshold, columns, n_kept, ws, index=None, n=None):
        n = xyz.shape[0] if n is None else n
        assert columns == [] and xyz.shape[0] == n and xyz.dtype == torch.float32
        s = fake_sdf(xyz)[:, 0]
        keep = torch.nonzero(s.abs() < torch.tensor(threshold, dtype=torch.float32)).view(-1)
        index[:keep.numel()] = keep
        n_kept[0] = keep.numel()
        calls.append((n, threshold))

    monkeypatch.setattr(cabi, "sdf_outlier_filter", op)
    return calls


@pytest.mark.parametrize("N", [1, 2, B - 1, B, B + 1, 2 * B, 2 * B + 1, 3 * B + 7])
def test_chunk_loop_evaluates_every_row_but_the_last(N):
    assert evaluated_rows(N, B) == list(range(N - 1))
    for b in (1, 2, B, 1_638_400):
        assert evaluated_rows(N, b) == list(range(N - 1))
        # the rows the twin evaluates: all of them but the only row of a one-row chunk
        n = SD.outlier_rows(N, b)
        one_row = [i for i in range(0, N, b) if min(i + b, N - 1) - i == 1]
        assert list(range(n)) == [r for r in evaluated_rows(N, b) if r not in one_row]


@pytest.mark.parametrize("N", [1, 2, B - 1, B, B + 1, B + 2, 2 * B, 2 * B + 1, 3 * B + 7])
@pytest.mark.parametrize("pattern", ["all", "none", "alternate", "random"])
def test_rule_equals_the_replay(N, pattern, host_operator):
    g = torch.Generator().manual_seed(N)
    keep = {"all": torch.ones(N, dtype=torch.bool), "none": torch.zeros(N, dtype=torch.bool),
            "alternate": torch.arange(N) % 2 == 0, "random": torch.rand(N, generator=g) < 0.6}[pattern]
    pack = make_pack(N, N, keep)
    thr = SD.outlier_threshold(2000, 30000, 0.6, 0.05)
    kept = rule(pack["xyz"], thr)
    try:
        ref = replay(pack, thr, B)
    except (RuntimeError, IndexError, ValueError):  # c10::Error in the reference's libtorch
        # the reference throws only when a chunk keeps exactly one row (squeeze() makes it 0-d): among several rows, the twin keeps it;
        # as the only row of its chunk, the twin drops it as the reference does where it does not throw
        chunks = [(i, min(i + B, N - 1)) for i in range(0, N, B)]
        ones = [(i, e) for i, e in chunks if int(((kept >= i) & (kept < e)).sum()) == 1]
        dropped_alone = [(i, e) for i, e in chunks if e - i == 1 and bool(fake_sdf(pack["xyz"][i:e]).abs()[0, 0] >= thr)]
        assert ones or dropped_alone
        ref = None
    if ref is not None:
        assert torch.equal(ref["xyz"], pack["xyz"][kept])
    # the twin: gate, n = N - 1, index_select of every field on the host
    out, count = SD.remove_outliers(_FakeNet(), pack, 2000, 30000, truncated_dis=0.6, outlier_dist=0.05, interval=2000, vis_batch_pt_num=B)
    assert host_operator[-1][0] == SD.outlier_rows(N, B) and count == kept.numel()
    for k, v in pack.items():
        assert torch.equal(out[k], v.index_select(0, kept)), k
        if ref is not None:
            assert torch.equal(out[k], ref[k]), k


def test_single_kept_row_in_a_chunk_raises_in_the_reference_and_is_kept(host_operator):
    N = 2 * B + 1
    keep = torch.zeros(N, dtype=torch.bool)
    keep[3] = True          # chunk 0 keeps exactly row 3
    keep[B:B + 4] = True    # chunk 1 keeps four rows
    pack = make_pack(N, 1, keep)
    with pytest.raises(RuntimeError):
        replay(pack, 0.25, B)
    out, count = SD.remove_outliers(_FakeNet(), pack, 4000, 5000, truncated_dis=0.6, outlier_dist=0.05, interval=2000, vis_batch_pt_num=B)
    assert count == 5 and torch.equal(out["xyz"], pack["xyz"][[3, B, B + 1, B + 2, B + 3]])


def test_one_row_chunk_keeps_nothing_in_the_reference(host_operator):
    """N = B + 2: the last chunk is row B alone; the reference drops it even when |sdf| < thr, and so does the twin."""
    N = B + 2
    pack = make_pack(N, 2, torch.ones(N, dtype=torch.bool))
    ref = replay(pack, 0.25, B)
    assert ref["xyz"].shape[0] == B
    out, count = SD.remove_outliers(_FakeNet(), pack, 4000, 5000, truncated_dis=0.6, outlier_dist=0.05, interval=2000, vis_batch_pt_num=B)
    assert count == B and all(torch.equal(out[k], ref[k]) for k in pack)


def test_empty_pack_raises_in_the_reference_and_stays_empty(host_operator):
    pack = make_pack(0, 0)
    with pytest.raises(ValueError):
        replay(pack, 0.25, B)
    out, count = SD.remove_outliers(_FakeNet(), pack, 2000, 5000, truncated_dis=0.6, outlier_dist=0.05, interval=2000, vis_batch_pt_num=B)
    assert count == 0 and all(v.shape[0] == 0 for v in out.values())


def test_gate(host_operator):
    pack = make_pack(50, 3)
    for it in (0, 1, 1999, 2001, 3000):
        out, count = SD.remove_outliers(_FakeNet(), pack, it, 5000, truncated_dis=0.6, outlier_dist=0.05, interval=2000, vis_batch_pt_num=B)
        assert out is pack and count == 50
    assert host_operator == []
    SD.remove_outliers(_FakeNet(), pack, 4000, 5000, truncated_dis=0.6, outlier_dist=0.05, interval=2000, vis_batch_pt_num=B)
    assert host_operator == [(49, SD.outlier_threshold(4000, 5000, 0.6, 0.05))]


# ---- the threshold ----
CPP = r"""
#include <cmath>
#include <cstdio>
#include <cstring>
#include <cstdint>
using namespace std;
int main() {
    int _iter, _total_iter;
    float k_truncated_dis;
    double k_outlier_dist;
    while (scanf("%d %d %a %la", &_iter, &_total_iter, &k_truncated_dis, &k_outlier_dist) == 4) {
        float iter_ratio = (float)_iter / _total_iter;
        auto tmp_outlier_dist = exp(log(k_truncated_dis) * (1 - iter_ratio) + log(k_outlier_dist) * iter_ratio);
        float t = (float)tmp_outlier_dist;  // what `tensor < double` compares against
        uint32_t u;
        uint64_t d;
        memcpy(&u, &t, 4);
        memcpy(&d, &tmp_outlier_dist, 8);
        printf("%u %llu\n", u, (unsigned long long)d);
    }
    return 0;
}
"""


def _sweep():
    rng = np.random.default_rng(0)
    rows = []
    for leaf in (0.2, 0.4, 0.05, 0.1):
        td = float(f32(3 * f32(leaf)))  # k_truncated_dis = 3 * k_leaf_size in fp32 (params.cpp:199)
        for od in (0.05, 0.02, 0.1):
            for total in (5000, 10000, 30000):
                its = sorted(set(list(range(0, total + 1, 2000)) + [1, 7, total - 1, total] + rng.integers(1, total, 20).tolist()))
                rows += [(it, total, td, od) for it in its]
    for _ in range(300):
        total = int(rng.integers(1, 40000))
        rows.append((int(rng.integers(0, total + 1)), total, float(f32(rng.uniform(0.01, 3.0))), float(rng.uniform(0.001, 1.0))))
    return rows


def test_threshold_matches_the_compiled_expression(tmp_path):
    src, exe = tmp_path / "thr.cpp", tmp_path / "thr"
    src.write_text(CPP)
    subprocess.check_call(["/usr/bin/g++", "-O3", "-fPIC", str(src), "-o", str(exe)])  # the reference's CMake flags
    rows = _sweep()
    inp = "".join(f"{it} {tot} {float(td).hex()} {od.hex()}\n" for it, tot, td, od in rows)
    out = subprocess.run([str(exe)], input=inp, capture_output=True, text=True, check=True).stdout.split("\n")
    n_rounded = 0
    for (it, tot, td, od), line in zip(rows, out):
        u, d = (int(v) for v in line.split())
        got = SD.outlier_threshold(it, tot, td, od)
        assert struct.unpack("<I", struct.pack("<f", got))[0] == u, (it, tot, td, od)
        tmp = struct.unpack("<d", struct.pack("<Q", d))[0]
        n_rounded += tmp != got
        # the fp32 threshold and the reference's double decide the same fp32 values, including the neighbours of the threshold
        t = torch.from_numpy(np.array([np.nextafter(f32(got), f32(0)), got, np.nextafter(f32(got), f32(np.inf))], f32))
        assert torch.equal(t < tmp, t < got) and torch.equal(t < got, torch.tensor([True, False, False]))
    assert n_rounded > 0.9 * len(rows)  # the double is almost never an fp32 value: the rounding is real
    # the shipped configs' end points: leaf 0.2 -> 0.6 at the start of a stage, outlier_dist at its end
    assert SD.outlier_threshold(0, 30000, float(f32(0.6)), 0.05) == float(f32(0.6))
    assert SD.outlier_threshold(30000, 30000, float(f32(0.6)), 0.05) == float(f32(0.05))


def test_comparison_against_a_double_is_in_fp32():
    """`tensor < double` rounds the scalar to the tensor's fp32 first (also checked on CUDA in test_gpu_outlier.py)."""
    v = f32(0.1)
    assert not bool((torch.tensor([v]) < float(v) + 1e-12)[0])
    assert bool((torch.tensor([v], dtype=torch.float64) < float(v) + 1e-12)[0])
