"""Times the joint stage (gstrain.GsTrainer, DESIGN 7o) on the box room at Replica's 1200x680, with splats from the SDF mesh
(gs_init.neural_gs_init after a short SdfTrainer stage), for each SH degree in --sh:

  color_init_s   the colour-initialisation epoch (one iteration per training frame)
  first_ms       steady-state ms per joint iteration in the first half (densification callback and its NaN-prune read every iteration)
  second_ms      the same in the second half (no callback)
  stage_s        the whole stage (colour init + --iters joint iterations, at least 2,000 per half by default), host clock with a final sync
  alternated     a second run of the stage in which windows of --window iterations alternate between GsTrainer.step and the same
                 operators driven the reference's way (tests/gs_train_replay.host_step: .item() reads of the sample std and the ray count,
                 host-scalar sampler and SDF sites, .item() on every logged value, the sample std taken in torch, the densification
                 callback's NaN prune read at once; the frame sent from pageable host memory): median ms per iteration of each driver in
                 each half

Frames live in pinned host memory (one asynchronous copy per iteration). Prints one JSON line per SH degree with the GPU's name and power
limit read in the same run.

--options instead times what the render background and the image mask cost: two trainers from the same SDF stage and splats, one with
the defaults and one with bck_color=1 and a mask (a quarter of the frame masked out), run second-half joint iterations (no densification,
so the splat count stays put) in alternating windows of --window iterations; prints the median and the spread (min, max) of the ms per
iteration of each.

  python tools/gs_train_bench.py [--sh 0,3] [--iters 4000] [--frames 60] [--window 50] [--rounds 4] [--options]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "gs-sdf_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from gssdf_b200 import gs_init as GI  # noqa: E402
from gssdf_b200 import gstrain as GT  # noqa: E402
from gssdf_b200 import nsdf as NS  # noqa: E402
from gssdf_b200 import octree as OT  # noqa: E402
from gssdf_b200 import scene as S  # noqa: E402
from gssdf_b200 import sdf as SD  # noqa: E402
import gs_train_replay as RP  # noqa: E402

LEAF, BCE_SIGMA = 0.05, 0.01  # config/replica/replica.yaml
W, H = 1200, 680
f32 = np.float32


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def poses(n, seed):
    rng = np.random.default_rng(seed)
    c2w = np.zeros((n, 4, 4), np.float32)
    for i in range(n):
        yaw, pitch = rng.uniform(0, 2 * math.pi), rng.uniform(-0.5, 0.5)
        f = np.array([math.cos(pitch) * math.cos(yaw), math.cos(pitch) * math.sin(yaw), math.sin(pitch)])
        right = np.cross(f, [0.0, 0.0, 1.0])
        right /= np.linalg.norm(right)
        c2w[i, :3, :3] = np.stack([right, np.cross(f, right), f], 1)
        c2w[i, :3, 3] = rng.uniform(-0.5, 0.5, 3) * S.BOX
        c2w[i, 3, 3] = 1.0
    return torch.from_numpy(c2w)


def ev_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sh", default="0,3")
    ap.add_argument("--iters", type=int, default=4000)
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--sdf-iters", type=int, default=200)
    ap.add_argument("--window", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--options", action="store_true", help="time bck_color=1 + a mask against the defaults")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    pack = S.box_room_pack(dev, 120, ds_pt_num=2000, seed=0)  # the depth pack of the GPU tests (its resolution does not enter the render)
    tree, frame, _ = OT.build_occ_map(pack["xyz"], pack["depth"], 0.01, 100.0, 14.0, LEAF)
    pos = np.asarray(frame["origin"], f32)
    lo = tuple(float(f32(pos[k] + f32(frame["xyz_min_M"][k]))) for k in range(3))
    hi = tuple(float(f32(pos[k] + f32(frame["xyz_max_M"][k]))) for k in range(3))
    margin = (tuple(float(f32(f32(v) + f32(0.5 * LEAF))) for v in frame["xyz_min_M"]),
              tuple(float(f32(f32(v) - f32(0.5 * LEAF))) for v in frame["xyz_max_M"]))
    c2w = poses(args.frames, 1)
    fx = W / 2.0
    imgs_dev = S.box_room_color(c2w.to(dev), fx, fx, (W - 1) / 2.0, (H - 1) / 2.0, W, H)
    imgs = imgs_dev.cpu().pin_memory()
    imgs_pageable = imgs_dev.cpu()
    del imgs_dev
    K = torch.tensor([[fx, 0, (W - 1) / 2.0], [0, fx, (H - 1) / 2.0], [0, 0, 1.0]])
    info = gpu_info()
    def trainer(sh, **kw):
        net = SD.SdfNet(dev, origin=frame["origin"], map_size=frame["map_size"], bce_isigma=1.0 / BCE_SIGMA, seed=1342)
        sdf = NS.SdfTrainer(net, tree, pack, args.sdf_iters, leaf_size=LEAF, bce_sigma=BCE_SIGMA, xyz_min=lo, xyz_max=hi, seed=5,
                            outlier_remove=True)
        sdf.run()
        sp, _ = GI.neural_gs_init(tree, sdf.write_back(), margin, LEAF, vis_batch_pt_num=1_638_400, sh_degree=sh,
                                  spatial_scale=0.5 * frame["inner_map_size"], inner_map_size=frame["inner_map_size"],
                                  map_origin=frame["origin"], sky=True, generator=torch.Generator(dev).manual_seed(0))
        n0 = int(sp["anchors"].shape[0])
        return GT.GsTrainer(sdf, sp, c2w, K, imgs, capacity=16 * n0, spatial_scale=0.5 * frame["inner_map_size"], gs_iter_step=args.iters,
                            sh_degree=sh, outlier_remove=True, **kw), n0

    w, half = args.window, args.iters // 2
    if args.options:
        mask = torch.ones(H, W, dtype=torch.bool, device=dev)
        mask[H // 4:3 * H // 4, W // 4:3 * W // 4] = False
        for sh in [int(s) for s in args.sh.split(",")]:
            runs = dict(defaults=trainer(sh)[0], bck_color_1_mask=trainer(sh, bck_color=1, mask=mask)[0])
            for G in runs.values():
                G.run_color_init()
                G.start_rates()
            ms = {k: [] for k in runs}
            for r in range(2 * args.rounds + 1):
                for k, G in runs.items():
                    i0 = half + r * w
                    t = ev_ms(lambda G=G, i0=i0: [G.step(j) for j in range(i0, min(i0 + w, args.iters))]) / w
                    if r > 0:  # the first window of each is the warm-up
                        ms[k].append(t)
            stat = lambda v: dict(median=round(float(np.median(v)), 3), min=round(min(v), 3), max=round(max(v), 3))
            print(json.dumps({"sh_degree": sh, "W": W, "H": H, "frames": args.frames, "splats": {k: G.T.N_live for k, G in runs.items()},
                              "window": w, "windows": 2 * args.rounds, **{k + "_ms": stat(v) for k, v in ms.items()}, "gpu": info}), flush=True)
            del runs
            torch.cuda.empty_cache()
        return
    for sh in [int(s) for s in args.sh.split(",")]:
        G, n0 = trainer(sh)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        color_ms = ev_ms(G.run_color_init)
        G.start_rates()

        def windows(start, stop):
            """ms per iteration of consecutive windows of w iterations over [start, stop); the first window is the warm-up"""
            out, i = [], start
            while i < stop:
                n = min(w, stop - i)
                ms = ev_ms(lambda i0=i, n_=n: [G.step(j) for j in range(i0, i0 + n_)]) / n
                if i > start:
                    out.append(ms)
                i += n
            return out
        first = windows(0, half)
        second = windows(half, args.iters)
        torch.cuda.synchronize()
        stage_s = time.perf_counter() - t0
        N_live = G.T.N_live
        del G
        torch.cuda.empty_cache()
        # the alternated run: even windows GsTrainer.step on pinned frames, odd windows the reference's way on pageable frames
        G, _ = trainer(sh)
        G.run_color_init()
        G.start_rates()
        alt = {("ours", 0): [], ("host", 0): [], ("ours", 1): [], ("host", 1): []}
        i, k = 0, 0
        while i < args.iters:
            n = min(w, (half if i < half else args.iters) - i)
            host = k % 2 == 1
            G.images = imgs_pageable if host else imgs
            ms = ev_ms(lambda i0=i, n_=n: [(RP.host_step(G, j) if host else G.step(j)) for j in range(i0, i0 + n_)]) / n
            if k >= 2 and i != half and i != half + w:  # skip the warm-up pair and the first pair after the switch of halves
                alt[("host" if host else "ours", int(i >= half))].append(ms)
            i += n
            k += 1
        med = lambda v: round(float(np.median(v)), 3) if v else None
        print(json.dumps({"sh_degree": sh, "W": W, "H": H, "frames": args.frames, "iters": args.iters, "splats_start": n0, "splats_end": N_live,
                          "color_init_s": round(color_ms / 1e3, 3), "first_ms": med(first), "second_ms": med(second), "stage_s": round(stage_s, 2),
                          "alternated_first_ours_ms": med(alt[("ours", 0)]), "alternated_first_host_ms": med(alt[("host", 0)]),
                          "alternated_second_ours_ms": med(alt[("ours", 1)]), "alternated_second_host_ms": med(alt[("host", 1)]),
                          "gpu": info}), flush=True)
        del G
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
