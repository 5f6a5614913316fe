"""Times what training on several cameras costs per joint iteration (gstrain.GsTrainer, DESIGN 7q), on the box room with splats from the
SDF mesh (gs_init.neural_gs_init after a short SdfTrainer stage, about 200 k splats at SH degree 0):

  one_size     --frames float frames at 1200x680 with one K (today's call), in pinned host memory
  mixed_size   the same poses on three cameras of similar pixel counts and different intrinsics, frame i on camera i % 3:
               1200x680, 1024x800 and 1360x600 (816 000, 819 200 and 816 000 pixels), float frames in pinned host memory
  u8_pinned    the one-size frames as an 8-bit FramesU8 store in pinned host memory (one frame's bytes copied per iteration and
               expanded on the device)
  u8_device    the same store on the device

Each trainer runs its own SDF stage, colour initialisation and the rate set-up; then windows of --window second-half joint iterations
(no densification callback, so the splat count stays put) alternate between the trainers for --rounds rounds after one warm-up round.
Prints one JSON line with the median and the spread (min, max) of the ms per iteration of each, the splat counts, and the GPU's name
and power limit read in the same run.

  python tools/multicam_train_bench.py [--iters 4000] [--frames 60] [--window 50] [--rounds 4] [--sh 0]
"""
import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "gs-sdf_b200"))

from gssdf_b200 import gs_init as GI  # noqa: E402
from gssdf_b200 import gstrain as GT  # noqa: E402
from gssdf_b200 import nsdf as NS  # noqa: E402
from gssdf_b200 import octree as OT  # noqa: E402
from gssdf_b200 import scene as S  # noqa: E402
from gssdf_b200 import sdf as SD  # noqa: E402

LEAF, BCE_SIGMA = 0.05, 0.01  # config/replica/replica.yaml
CAMERAS = [(1200, 680), (1024, 800), (1360, 600)]
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


def K_of(W, H, c):
    f = W / 2.0 * (1.0, 1.08, 0.93)[c]
    return torch.tensor([[f, 0, (W - 1) / 2.0 + 2 * c], [0, f, (H - 1) / 2.0 - c], [0, 0, 1.0]], dtype=torch.float32)


def ev_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sh", type=int, default=0)
    ap.add_argument("--iters", type=int, default=4000)
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--sdf-iters", type=int, default=200)
    ap.add_argument("--window", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=4)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    pack = S.box_room_pack(dev, 120, ds_pt_num=2000, seed=0)
    tree, frame, _ = OT.build_occ_map(pack["xyz"], pack["depth"], 0.01, 100.0, 14.0, LEAF)
    pos = np.asarray(frame["origin"], f32)
    lo = tuple(float(f32(pos[k] + f32(frame["xyz_min_M"][k]))) for k in range(3))
    hi = tuple(float(f32(pos[k] + f32(frame["xyz_max_M"][k]))) for k in range(3))
    margin = (tuple(float(f32(f32(v) + f32(0.5 * LEAF))) for v in frame["xyz_min_M"]),
              tuple(float(f32(f32(v) - f32(0.5 * LEAF))) for v in frame["xyz_max_M"]))
    n = args.frames
    c2w = poses(n, 1)
    W0, H0 = CAMERAS[0]
    K0 = K_of(W0, H0, 0)
    one = S.box_room_color(c2w.to(dev), float(K0[0, 0]), float(K0[1, 1]), float(K0[0, 2]), float(K0[1, 2]), W0, H0)
    u8 = [(one[i] * 255).round().to(torch.uint8).cpu() for i in range(n)]
    one = one.cpu().pin_memory()
    Ks, mixed = [], []
    for i in range(n):
        c = i % 3
        W, H = CAMERAS[c]
        K = K_of(W, H, c)
        Ks.append(K)
        mixed.append(S.box_room_color(c2w[i:i + 1].to(dev), float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]), W, H)[0]
                     .cpu().pin_memory())
    configs = dict(one_size=(K0, one), mixed_size=(torch.stack(Ks), mixed), u8_pinned=(K0, GT.FramesU8.pack(u8, pin=True)),
                   u8_device=(K0, GT.FramesU8.pack(u8, device=dev)))
    info = gpu_info()

    def trainer(K, images):
        net = SD.SdfNet(dev, origin=frame["origin"], map_size=frame["map_size"], bce_isigma=1.0 / BCE_SIGMA, seed=1342)
        sdf = NS.SdfTrainer(net, tree, pack, args.sdf_iters, leaf_size=LEAF, bce_sigma=BCE_SIGMA, xyz_min=lo, xyz_max=hi, seed=5,
                            outlier_remove=True)
        sdf.run()
        sp, _ = GI.neural_gs_init(tree, sdf.write_back(), margin, LEAF, vis_batch_pt_num=1_638_400, sh_degree=args.sh,
                                  spatial_scale=0.5 * frame["inner_map_size"], inner_map_size=frame["inner_map_size"],
                                  map_origin=frame["origin"], sky=True, generator=torch.Generator(dev).manual_seed(0))
        return GT.GsTrainer(sdf, sp, c2w, K, images, capacity=16 * int(sp["anchors"].shape[0]), spatial_scale=0.5 * frame["inner_map_size"],
                            gs_iter_step=args.iters, sh_degree=args.sh, outlier_remove=True)

    runs = {k: trainer(*v) for k, v in configs.items()}
    for G in runs.values():
        G.run_color_init()
        G.start_rates()
    w, start = args.window, args.iters // 2
    ms = {k: [] for k in runs}
    for r in range(args.rounds + 1):
        for k, G in runs.items():
            i0 = start + r * w
            t = ev_ms(lambda G=G, i0=i0: [G.step(j) for j in range(i0, min(i0 + w, args.iters))]) / w
            if r > 0:  # the first window of each is the warm-up
                ms[k].append(t)
    for G in runs.values():
        G.histories()  # raises on a sampler overflow
    stat = lambda v: dict(median=round(float(np.median(v)), 3), min=round(min(v), 3), max=round(max(v), 3))
    print(json.dumps({"sh_degree": args.sh, "cameras": CAMERAS, "frames": n, "splats": {k: G.T.N_live for k, G in runs.items()},
                      "window": w, "windows": args.rounds, **{k + "_ms": stat(v) for k, v in ms.items()},
                      "frame_store_MB": dict(float=round(4 * 3 * W0 * H0 * n / 2 ** 20, 1), u8=round(3 * W0 * H0 * n / 2 ** 20, 1)),
                      "gpu": info}), flush=True)


if __name__ == "__main__":
    main()
