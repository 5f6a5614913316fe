"""f-13 without a GPU: the scalar rules of nsdf_train / sdf_train_callback that gssdf_sdf_adapt and SdfTrainer apply -- the samples-per-ray
EMA, the ray count, the initial state and the learning-rate schedule -- restated in numpy (gssdf_b200.nsdf) and compared bit for bit with the
reference's C++ expressions compiled with g++ -O3 (its CMake flags); the batch draw's index rule against torch's CPU
`(rand * N).to(kLong).clamp(0, N - 1)`; and the argument errors of the five f-13 entry points, which return before any CUDA call."""
import ctypes
import struct
import subprocess

import numpy as np
import pytest
import torch

from gssdf_b200 import _lib
from gssdf_b200 import nsdf as NS

f32 = np.float32
INT_LIMIT = 2147483648.0  # (int)q is defined for q < 2^31


def bits(v):
    return struct.unpack("<I", struct.pack("<f", float(v)))[0]


# nsdf_train :298-299 and :324-330 with params.cpp:203-204, statement for statement in the reference's types (params.h:34-36). Where
# (int)(k_batch_pt_num / k_sample_pts_per_ray) would be undefined (q >= 2^31: a long run of zero-sample iterations), the line is flagged
# and the trajectory continues with (int)k_batch_pt_num, the value the min() takes wherever the conversion is defined and q is that large.
CPP_RAYS = r"""
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <cstdint>
using namespace std;
float k_batch_pt_num, k_sample_pts_per_ray;
int k_batch_num, k_batch_ray_num;
static unsigned fb(float f) { unsigned u; memcpy(&u, &f, 4); return u; }
int main() {
    int n_steps;
    while (scanf("%a %d", &k_batch_pt_num, &n_steps) == 2) {
        k_batch_ray_num = k_batch_pt_num;
        k_batch_num = k_batch_ray_num;
        k_sample_pts_per_ray = k_batch_pt_num / (float)k_batch_num;
        printf("%u %d 0\n", fb(k_sample_pts_per_ray), k_batch_num);
        for (int s = 0; s < n_steps; ++s) {
            long long v;
            if (scanf("%lld", &v) != 1) return 1;
            float pt_n = v;
            float sample_pts_per_ray = pt_n / (float)k_batch_num;
            k_sample_pts_per_ray = k_sample_pts_per_ray * 0.9 + sample_pts_per_ray * 0.1;
            float q = k_batch_pt_num / k_sample_pts_per_ray;
            int ub = !(q < 2147483648.0f);
            if (ub) k_batch_num = (int)k_batch_pt_num;
            else k_batch_num = min((int)(k_batch_pt_num / k_sample_pts_per_ray), (int)k_batch_pt_num);
            printf("%u %d %d\n", fb(k_sample_pts_per_ray), k_batch_num, ub);
        }
    }
    return 0;
}
"""

# sdf_train_callback :542,550-551
CPP_LR = r"""
#include <cstdio>
#include <cstring>
int main() {
    int _iter, _total_iter;
    float k_lr, k_lr_end;
    while (scanf("%d %d %a %a", &_iter, &_total_iter, &k_lr, &k_lr_end) == 4) {
        float iter_ratio = (float)_iter / _total_iter;
        float lr = k_lr * (1 - iter_ratio) + k_lr_end * iter_ratio;
        unsigned u;
        memcpy(&u, &lr, 4);
        printf("%u\n", u);
    }
    return 0;
}
"""


def _compile(tmp_path, name, src):
    c, exe = tmp_path / f"{name}.cpp", tmp_path / name
    c.write_text(src)
    subprocess.check_call(["/usr/bin/g++", "-O3", "-fPIC", str(c), "-o", str(exe)])
    return exe


def _trajectories():
    """(batch_pt_num, [pt_n per iteration]): the stage's regimes, sample counts 0 .. 1e6, long runs of zero-sample iterations (the EMA
    decays through the denormals to 0 and q passes 2^31), and recoveries after them."""
    rng = np.random.default_rng(0)
    out = []
    for bpn in (32768.0, 1000.0, 65536.0, 12345.0, 1.0, 3.0):
        out.append((bpn, rng.integers(0, 1_000_001, 300).tolist()))
        out.append((bpn, [0] * 1200 + rng.integers(0, 50_000, 50).tolist()))
        out.append((bpn, (rng.integers(20_000, 45_000, 200)).tolist() + [0] * 150 + [1, 2, 3, 10**6, 0, 7]))
        out.append((bpn, [int(bpn) * k for k in (0, 1, 2, 5, 10, 30, 100)] * 20))
    out.append((32768.0, [0, 1, 10**6, 10**6 - 1, 999_999, 2**24, 2**24 + 1, 123_457] * 30))
    return out


def test_adapt_rules_match_the_compiled_expressions(tmp_path):
    exe = _compile(tmp_path, "rays", CPP_RAYS)
    traj = _trajectories()
    inp = "".join(f"{float(f32(b)).hex()} {len(p)}\n" + "".join(f"{v}\n" for v in p) for b, p in traj)
    lines = iter(subprocess.run([str(exe)], input=inp, capture_output=True, text=True, check=True).stdout.split("\n"))
    n_ub = n_steps = 0
    for b, seq in traj:
        ppr, n = NS.initial_state(b)
        u, r, _ = (int(v) for v in next(lines).split())
        assert (bits(ppr), n) == (u, r), ("initial", b)
        for s, pt in enumerate(seq):
            ppr, n = NS.adapt_rays(ppr, n, pt, b)
            u, r, ub = (int(v) for v in next(lines).split())
            assert bits(ppr) == u, (b, s, pt)
            assert n == r, (b, s, pt)  # in the undefined region the restatement gives (int)batch_pt_num, as the guarded C++ line does
            n_ub += ub
            n_steps += 1
    assert n_ub > 1000  # the INT_MAX edge is exercised ...
    assert n_steps - n_ub > 4000  # ... and so is the defined region


def test_ray_count_edges():
    # the min is taken in float: the float just below 2^31 still converts; 2^31 itself would not, and gives the cap
    b = f32(32768)
    ppr_edge = f32(b / f32(np.nextafter(f32(INT_LIMIT), f32(0))))
    assert NS.adapt_rays(ppr_edge / f32(0.9), 32768, 0, b)[1] == 32768
    assert NS.adapt_rays(f32(0), 32768, 0, b) == (f32(0), 32768)
    # a batch of exactly batch_pt_num samples per ray: one ray
    ppr, n = NS.initial_state(32768.0)
    assert (ppr, n) == (f32(1), 32768)
    for _ in range(400):
        ppr, n = NS.adapt_rays(ppr, n, n * 10, 32768.0)
    assert n in (3276, 3277) and abs(float(ppr) - 10.0) < 1e-3  # settles where batch_pt_num / pts_per_ray puts it


def _lr_rows():
    rng = np.random.default_rng(1)
    rows = []
    for total in (5000, 30000, 1, 7, 10000):
        its = sorted(set(list(range(0, total + 1, max(total // 50, 1))) + [0, 1, total - 1, total]))
        rows += [(it, total, 5e-3, 1e-4) for it in its]
    for _ in range(500):
        total = int(rng.integers(1, 50_000))
        rows.append((int(rng.integers(0, total + 1)), total, float(f32(rng.uniform(1e-5, 1e-1))), float(f32(rng.uniform(1e-6, 1e-2)))))
    return rows


def test_learning_rate_schedule_matches_the_compiled_expression(tmp_path):
    exe = _compile(tmp_path, "lr", CPP_LR)
    rows = _lr_rows()
    inp = "".join(f"{it} {tot} {float(f32(a)).hex()} {float(f32(b)).hex()}\n" for it, tot, a, b in rows)
    out = subprocess.run([str(exe)], input=inp, capture_output=True, text=True, check=True).stdout.split()
    for (it, tot, a, b), u in zip(rows, out):
        assert bits(NS.lr_at(it, tot, a, b)) == int(u), (it, tot, a, b)
    assert NS.lr_at(0, 5000, 5e-3, 1e-4) == float(f32(5e-3)) and NS.lr_at(5000, 5000, 5e-3, 1e-4) == float(f32(1e-4))


@pytest.mark.parametrize("N", [1, 2, 3, 1000, 2**24 - 1, 2**24, 2**24 + 1, 2**24 + 3, 2**25 + 1, 10_000_003, 2**31 + 5])
def test_ray_index_rule_equals_torch(N):
    one = f32(1)
    near_one = [np.nextafter(one, f32(0))]
    for _ in range(40):
        near_one.append(np.nextafter(near_one[-1], f32(0)))
    rng = np.random.default_rng(N % 1000)
    r = np.concatenate([np.array(near_one, f32), np.array([0.0, 1e-30, 0.5, 0.25], f32), rng.random(4000, dtype=f32)])
    want = (torch.from_numpy(r) * N).to(torch.long).clamp(0, N - 1).numpy()
    got = NS.ray_index(r, N)
    assert np.array_equal(got, want)
    if float(f32(N)) > N:  # N rounds up in fp32: values next to 1 land on N itself and are clamped
        assert int(want[0]) == N - 1


# ---- argument errors (no CUDA call is made before these checks) ----
def _err():
    return _lib.lib().gssdf_last_error()


def test_argument_errors_of_the_f13_entry_points():
    L = _lib.lib()
    p = ctypes.c_void_p(256)  # a non-null pointer that is never dereferenced on these paths
    # gssdf_sdf_ray_batch
    assert L.gssdf_sdf_ray_batch(None, None) == -1 and b"null args" in _err()
    full = dict(N=10, ray_cap=4, rand=p, n_rays=p, origin=p, direction=p, depth=p, xyz=p, origin_out=p, direction_out=p, depth_out=p, xyz_out=p)
    for k, v, msg in (("N", 0, b"at least one row"), ("ray_cap", -1, b"negative ray_cap"), ("n_rays", None, b"n_rays"),
                      ("rand", None, b"rand and the pack"), ("xyz", None, b"rand and the pack"), ("depth_out", None, b"null output")):
        a = _lib.make_args("gssdf_sdf_ray_batch_args", **{**full, k: v})
        assert L.gssdf_sdf_ray_batch(ctypes.byref(a), None) == -1, k
        assert msg in _err(), (k, _err())
    # gssdf_sdf_adapt
    assert L.gssdf_sdf_adapt(None, None) == -1 and b"null args" in _err()
    full = dict(state=p, y1=p, y1_cap=8, n_samples=p, bce_sigma=0.01, bce_isigma=100.0, batch_pt_num=32768.0, update_rays=1)
    for k, v, msg in (("state", None, b"state and n_samples"), ("n_samples", None, b"state and n_samples"), ("y1", None, b"y1 is required"),
                      ("y1_cap", -1, b"y1 is required"), ("bce_sigma", 0.0, b"bce_sigma"), ("bce_sigma", float("nan"), b"bce_sigma"),
                      ("batch_pt_num", 0.5, b"batch_pt_num"), ("batch_pt_num", INT_LIMIT, b"batch_pt_num")):
        a = _lib.make_args("gssdf_sdf_adapt_args", **{**full, k: v})
        assert L.gssdf_sdf_adapt(ctypes.byref(a), None) == -1, k
        assert msg in _err(), (k, _err())
    # gssdf_sdf_sample_rays_dev: the checks of gssdf_sdf_sample_rays
    assert L.gssdf_sdf_sample_rays_dev(None, p, p, None) == -1 and b"null args" in _err()
    a = _lib.make_args("gssdf_sdf_sample_rays_args", n_rays=-1)
    assert L.gssdf_sdf_sample_rays_dev(ctypes.byref(a), p, p, None) == -1 and b"negative size" in _err()
    a = _lib.make_args("gssdf_sdf_sample_rays_args", n_rays=4, voxel_sample_num=0)
    assert L.gssdf_sdf_sample_rays_dev(ctypes.byref(a), p, p, None) == -1 and b"bad sample counts" in _err()
    # gssdf_sdf_fwd_dev / gssdf_sdf_train_dev: the checks of gssdf_sdf_fwd / gssdf_sdf_train
    assert L.gssdf_sdf_fwd_dev(None, p, None) == -1 and b"null args" in _err()
    net = _lib.make_args("gssdf_sdf_net", n_levels=16, n_features_per_level=2, log2_hashmap_size=19, base_resolution=32, per_level_scale=2.0,
                         hidden_dim=64, n_hidden=3, table_half=p, mlp=p, mlp_mode=1, mlp_packed=p)
    a = _lib.make_args("gssdf_sdf_fwd_args", n=4, x=p, sdf=p, n_variants=3)
    a.net = net
    assert L.gssdf_sdf_fwd_dev(ctypes.byref(a), p, None) == -1 and b"n_variants" in _err()
    assert L.gssdf_sdf_train_dev(None, p, None) == -1 and b"null args" in _err()
    t = _lib.make_args("gssdf_sdf_train_args", n=4, x=p, n_variants=1)
    t.net = net
    t.net.mlp_mode = 0
    assert L.gssdf_sdf_train_dev(ctypes.byref(t), p, None) == -3 and b"mlp_mode 1 only" in _err()
    t.net.mlp_mode = 1
    t.n_variants = 5
    assert L.gssdf_sdf_train_dev(ctypes.byref(t), p, None) == -1 and b"n_variants" in _err()
    # the host-scalar call still rejects a non-positive delta; the device call leaves delta to the caller (sample_std >= bce_sigma > 0)
    t.n_variants, t.eikonal_mode, t.align_weight, t.sdf_variants = 7, 1, 0.1, None
    assert L.gssdf_sdf_train(ctypes.byref(t), None) == -1 and b"delta must be positive" in _err()
    t.eikonal_mode = 2
    assert L.gssdf_sdf_train_dev(ctypes.byref(t), p, None) == -1 and b"eikonal_mode" in _err()


def test_initial_device_state_layout():
    """new_adapt_state packs {sample_std, pts_per_ray, n_rays} as gssdf_sdf_adapt_state lays them out."""
    S = _lib.STRUCTS["gssdf_sdf_adapt_state"]
    assert ctypes.sizeof(S) == 16 and S.sample_std.offset == 0 and S.pts_per_ray.offset == 4 and S.n_rays.offset == 8
    ppr, n = NS.initial_state(32768.0)
    raw = np.zeros(4, np.int32)
    raw[:2] = np.array([0.01, ppr], f32).view(np.int32)
    raw[2] = n
    s = S.from_buffer_copy(raw.tobytes())
    assert s.sample_std == float(f32(0.01)) and s.pts_per_ray == 1.0 and s.n_rays == 32768
