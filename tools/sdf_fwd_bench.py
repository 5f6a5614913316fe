"""Timing and output dump of the tensor-core SDF forward (gssdf_sdf_fwd, mlp_mode 1) at the batch shapes of the training step.

    python tools/sdf_fwd_bench.py [--iters 200] [--dump out.npz]

Cases (bench.py 1080p-1M; capacities as GsSdfTrainer allocates them, live counts as the step census measured them, on the device):
  A     the align loss's offset forward on the ray samples: capacity 49152, 27300 live, 7 variants, skip_base_variant
  C     the same on the gated splat samples: capacity 1 M, 102500 live, 7 variants, skip_base_variant
  plain n_variants 1, sdf + y1, 40000 points
  feat  7 variants, sdf + y1 + feat, 20000 points
Inputs come from a fixed seed, so two builds of the library can be compared array by array (--dump, then np.array_equal). Outputs
start as NaN: rows a launch does not write stay NaN in both builds.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "gs-sdf_b200")]

import torch  # noqa: E402

from gssdf_b200 import cabi  # noqa: E402

CASES = {  # name: (capacity n, live rows or None, n_variants, skip_base_variant, y1, feat)
    "A": (49152, 27300, 7, True, False, False),
    "C": (1_000_000, 102500, 7, True, False, False),
    "plain": (40000, None, 1, False, True, False),
    "feat": (20000, None, 7, False, True, True),
}


def make_net(dev, seed=7, n_hidden=3):
    rng = np.random.default_rng(seed)
    n_params = cabi.sdf_table_params(cabi.sdf_net(torch.zeros(1, device=dev), torch.zeros(1, device=dev)))
    table = torch.from_numpy(rng.uniform(-0.5, 0.5, n_params).astype(np.float32)).to(dev)
    dims, ps = [32] + [64] * (1 + n_hidden) + [2], []
    for k, o in zip(dims[:-1], dims[1:]):
        b = 1 / np.sqrt(k)
        ps += [rng.uniform(-b, b, o * k), rng.uniform(-b, b, o)]
    mlp = torch.from_numpy(np.concatenate(ps).astype(np.float32)).to(dev)
    half = torch.empty(n_params, dtype=torch.float16, device=dev)
    cabi.sdf_table_to_half(table, half)
    probe = cabi.sdf_net(half, mlp, hidden_dim=64, n_hidden=n_hidden)
    packed = torch.empty(cabi.sdf_mlp_packed_bytes(probe), dtype=torch.uint8, device=dev)
    cabi.sdf_mlp_pack(probe, packed)
    return cabi.sdf_net(half, mlp, hidden_dim=64, n_hidden=n_hidden, mlp_mode=1, mlp_packed=packed), (half, mlp, packed)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--dump", help="write every output array of every case to this .npz")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    net, keep = make_net(dev)
    g = torch.Generator(dev).manual_seed(11)
    res, dump = {}, {}
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for name, (n, live, nv, skip, want_y1, want_feat) in CASES.items():
        x = torch.rand(n, 3, device=dev, generator=g) * 0.96 + 0.02
        n_live = torch.tensor([live], dtype=torch.int32, device=dev) if live is not None else None
        sdf = torch.full((n * nv,), float("nan"), device=dev)
        y1 = torch.full((n * nv,), float("nan"), device=dev) if want_y1 else None
        feat = torch.full((n * nv, 32), float("nan"), device=dev) if want_feat else None
        call = lambda: cabi.sdf_fwd(net, x, sdf, y1, feat, n_variants=nv, delta=0.01, n_live=n_live, skip_base_variant=skip)
        call()
        torch.cuda.synchronize()
        for k, v in (("sdf", sdf), ("y1", y1), ("feat", feat)):
            if v is not None:
                dump[f"{name}.{k}"] = v.cpu().numpy()
        for _ in range(10):
            call()
        s.record()
        for _ in range(args.iters):
            call()
        e.record()
        torch.cuda.synchronize()
        res[name] = s.elapsed_time(e) / args.iters * 1e3
        print(f"{name:6s} n={n:<8d} live={live if live is not None else n:<8} V={nv} skip_base={int(skip)}  {res[name]:8.1f} us/call")
    print(json.dumps({"device": torch.cuda.get_device_name(), "us_per_call": res, "iters": args.iters}))
    if args.dump:
        np.savez(args.dump, **dump)


if __name__ == "__main__":
    main()
