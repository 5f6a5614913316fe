"""Times the SDF pre-training stage (row f-13, DESIGN 7n) on the box room's depth pack:

  trainer   SdfTrainer: per iteration at the steady-state ray count, and the whole stage (--iters, 5000 in every shipped config)
  host      the same operators driven the reference's way (sdf_train_batch_iter / nsdf_train / sdf_train_callback): every iteration reads
            the sample std and the ray count back with .item(), draws the ray indices with a CPU torch.rand, indexes a CPU copy of the pack
            and sends the rays to the device with .to(device), and reads the sample count and mean(1 / isigma) back for the next iteration

for each pack size in --rows (2 M and 10 M rows by default). Prints one JSON line per pack with the GPU's name and power limit read in the
same run; --out also writes them to a file.

  python tools/nsdf_bench.py [--rows 2000000,10000000] [--iters 5000] [--steady 500] [--out results/nsdf_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "gs-sdf_b200"))

from gssdf_b200 import cabi  # noqa: E402
from gssdf_b200 import nsdf as NS  # noqa: E402
from gssdf_b200 import octree as OT  # noqa: E402
from gssdf_b200 import scene as S  # noqa: E402
from gssdf_b200 import sdf as SD  # noqa: E402

LEAF, BCE_SIGMA = 0.05, 0.01  # config/replica/replica.yaml
f32 = np.float32


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def room(dev, rows, seed=0):
    per_frame = 10_000
    pack = S.box_room_pack(dev, max(rows // per_frame, 1), ds_pt_num=per_frame, seed=seed)
    tree, frame, _ = OT.build_occ_map(pack["xyz"], pack["depth"], 0.01, 100.0, 14.0, LEAF)
    pos = np.asarray(frame["origin"], f32)
    lo = tuple(float(f32(pos[k] + f32(frame["xyz_min_M"][k]))) for k in range(3))
    hi = tuple(float(f32(pos[k] + f32(frame["xyz_max_M"][k]))) for k in range(3))
    return pack, tree, frame, lo, hi


def trainer(dev, pack, tree, frame, lo, hi, iters):
    net = SD.SdfNet(dev, origin=frame["origin"], map_size=frame["map_size"], bce_isigma=1.0 / BCE_SIGMA)
    return NS.SdfTrainer(net, tree, pack, iters, leaf_size=LEAF, bce_sigma=BCE_SIGMA, xyz_min=lo, xyz_max=hi)


class HostDriven:
    """The same operators with the reference's host round trips (sdf_train_batch_iter :143-156, nsdf_train :324-330, callback :544-557)."""

    def __init__(self, T, pack):
        self.T = T
        self.cpu_pack = {k: v.cpu() for k, v in pack.items()}
        self.N = pack["xyz"].shape[0]
        self.s7 = torch.empty(7 * T.rs.cap, device=T.dev)
        self.y7 = torch.empty(7 * T.rs.cap, device=T.dev)
        self.ppr, self.n_rays = NS.initial_state(T.batch_pt_num)
        self.std = T.bce_sigma

    def step(self, i):
        T, rs, dev = self.T, self.T.rs, self.T.dev
        k = self.n_rays
        idx = (torch.rand(k) * self.N).to(torch.long).clamp(0, self.N - 1)  # CPU torch::rand
        rays = {key: v.index_select(0, idx).to(dev) for key, v in self.cpu_pack.items()}
        T.draw()
        rs.n, rs.std = k, self.std  # the sampler's host ray count and std
        rs.sample(rays["origin"], rays["direction"], rays["depth"].reshape(-1).contiguous(), rays["xyz"])
        rs.n = T.ray_cap
        cabi.sdf_fwd(T.net, rs.xyz, self.s7, self.y7, n_variants=7, delta=self.std, n_live=rs.counts)
        cabi.sdf_train(T.net, rs.xyz, 1, self.std, rs.ray_sdf, None, T.bce_isigma, 1.0, T.eik_w, 0.0, T.h_loss[i:i + 1], T.table_grad, T.mlp_grad,
                       None, n_live=rs.counts, eikonal_mode=1, align_weight=T.align_w, sdf_variants=self.s7)
        T.t += 1
        cabi.adam_step(T.params, T.grad, T.exp_avg, T.exp_avg_sq, T.sdf_groups(T.lr), T.t, eps=1e-15, zero_grads=True, table_half=T.table_half,
                       net=T.net, mlp_packed=T.mlp_packed)
        pt_n = int(rs.counts[0].item())  # point_samples.size(0)
        self.ppr, self.n_rays = NS.adapt_rays(self.ppr, self.n_rays, pt_n, T.batch_pt_num)
        if pt_n > 0:
            inv = 1.0 / (1 + torch.nn.functional.softplus(self.y7[:pt_n], beta=100) * T.bce_isigma)
            self.std = max(float(inv.mean().item()), T.bce_sigma)
        T.lr = NS.lr_at(i, T.iters, T.lr0, T.lr_end)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", default="2000000,10000000")
    ap.add_argument("--iters", type=int, default=5000)
    ap.add_argument("--steady", type=int, default=500, help="iterations timed per step after --warm")
    ap.add_argument("--warm", type=int, default=300)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("nsdf_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    gpu = gpu_info()
    results = []
    for rows in (int(r) for r in args.rows.split(",")):
        pack, tree, frame, lo, hi = room(dev, rows)
        res = dict(gpu=gpu, rows=int(pack["xyz"].shape[0]), iters=args.iters)
        for name in ("trainer", "host"):
            T = trainer(dev, pack, tree, frame, lo, hi, args.iters)
            drv = HostDriven(T, pack) if name == "host" else T
            timed(lambda: [drv.step(i) for i in range(args.warm)])
            per = timed(lambda: [drv.step(i) for i in range(args.warm, args.warm + args.steady)]) / args.steady
            T = trainer(dev, pack, tree, frame, lo, hi, args.iters)
            drv = HostDriven(T, pack) if name == "host" else T
            stage = timed(lambda: [drv.step(i) for i in range(args.iters)])
            n_rays = int(NS.read_state(T.adapt)[2]) if name == "trainer" else drv.n_rays
            res[name] = dict(ms_per_iter_steady=round(per * 1e3, 4), stage_s=round(stage, 3), final_n_rays=n_rays)
        res["stage_speedup"] = round(res["host"]["stage_s"] / res["trainer"]["stage_s"], 3)
        print(json.dumps(res), flush=True)
        results.append(res)
        del pack, tree
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(results, fh, indent=1)


if __name__ == "__main__":
    main()
