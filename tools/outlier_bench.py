"""Timing of gssdf_sdf_outlier_filter (sdf.remove_outliers on a device-resident pack, DESIGN 7m) against the reference's composition
(neural_mapping.cpp:563-590) on the same GPU: chunks of k_vis_batch_pt_num = 1,638,400 rows through SdfNet.get_sdf, `abs() < thr`,
nonzero(), .cpu(), cat and a host index_select of a CPU-resident pack. Needs a CUDA device.

Packs have the trainer's four fields, origin [N,3], direction [N,3], depth [N,1], xyz [N,3] (40 B/row), at 1 M rows (the COLMAP configs'
max_pt_num), 5 M (oxford) and 10 M (fast_livo). Clouds: the 300 m outdoor scene of tools/octree_build_bench.py and the box room's walls
with 1 cm noise and 1 % outliers in free space, both evaluated by the fitted box-room net (scene.box_room_sdf_net) at the threshold of
iteration 4000 of 5000 with leaf 0.2 (0.098 m). The operator is timed with CUDA events (median of --reps calls after a warm-up), split
into its SDF part (gssdf_sdf_fwd alone on the same rows) and the rest (selection + gather = operator - SDF); the composition is timed on
the host clock around the whole branch. The outputs are compared byte for byte. Prints one JSON line per size and cloud, and the GPU's
name and power limit.

usage: python tools/outlier_bench.py [--reps 5] [--sizes 1000000,5000000,10000000]"""
import argparse
import importlib.util
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "gs-sdf_b200")]

import torch  # noqa: E402

from gssdf_b200 import cabi  # noqa: E402
from gssdf_b200 import scene as S  # noqa: E402
from gssdf_b200 import sdf as SD  # noqa: E402

_spec = importlib.util.spec_from_file_location("octree_build_bench", os.path.join(ROOT, "tools", "octree_build_bench.py"))
OB = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(OB)

B = 1_638_400
HBM = 3.35e12
IT, TOTAL, TD, OD = 4000, 5000, float(np.float32(3 * np.float32(0.2))), 0.05


def box_cloud(n, g, dev):
    """Wall points of the box room with 1 cm noise, and 1 % outliers anywhere in the room."""
    k = n // 100
    b = torch.as_tensor(S.BOX, dtype=torch.float32, device=dev)
    face = torch.randint(0, 6, (n - k,), device=dev, generator=g)
    p = (torch.rand(n - k, 3, device=dev, generator=g) * 2 - 1) * b
    ax = face // 2
    sgn = (face % 2) * 2 - 1
    p[torch.arange(n - k, device=dev), ax] = sgn.float() * b[ax]
    p += torch.randn(n - k, 3, device=dev, generator=g) * 0.01
    out = (torch.rand(k, 3, device=dev, generator=g) * 2 - 1) * b
    return torch.cat([p, out])[torch.randperm(n, device=dev, generator=g)].contiguous()


def make_pack(xyz, g):
    n = xyz.shape[0]
    origin = (torch.rand(n, 3, device=xyz.device, generator=g) * 2 - 1)
    d = xyz - origin
    depth = d.norm(dim=1, keepdim=True)
    return {"origin": origin, "direction": (d / depth).contiguous(), "depth": depth, "xyz": xyz}


def composition(net, pack_cpu, thr_double):
    """sdf_train_callback's outlier branch as the reference runs it."""
    train_pcl = pack_cpu["xyz"].view(-1, 3)
    point_num = train_pcl.shape[0]
    vec = []
    t_sdf = 0.0
    for i in range(0, point_num, B):
        end = min(i + B, point_num - 1)
        t0 = time.perf_counter()
        s = net.get_sdf(train_pcl.index_select(0, torch.arange(i, end)).to("cuda"))[0]
        torch.cuda.synchronize()
        t_sdf += time.perf_counter() - t0
        vec.append((s.abs() < thr_double).squeeze().nonzero().squeeze().cpu() + i)
    idx = torch.cat(vec, 0)
    return {k: v.index_select(0, idx) for k, v in pack_cpu.items()}, t_sdf


def ev_time(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sizes", default="1000000,5000000,10000000")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "outlier_bench needs a CUDA device"
    dev = torch.device("cuda:0")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": gpu}), flush=True)
    torch.manual_seed(0)
    net, _, _ = S.box_room_sdf_net(dev)
    ns = net._net(net.params_, net.decoder_)
    thr = SD.outlier_threshold(IT, TOTAL, TD, OD)
    m = SD._m()
    ratio = np.float32(IT) / np.float32(TOTAL)
    thr_double = m.exp(float(np.float32(m.logf(TD)) * (np.float32(1) - ratio)) + m.log(OD) * float(ratio))
    ws = cabi.Workspace(dev)
    for N in (int(s) for s in args.sizes.split(",")):
        for cloud in ("outdoor", "box_room"):
            g = torch.Generator(device=dev).manual_seed(N)
            xyz = OB.outdoor_cloud(N, g, dev) if cloud == "outdoor" else box_cloud(N, g, dev)
            pack = make_pack(xyz, g)
            n = SD.outlier_rows(N, B)
            out = {k: torch.empty_like(v) for k, v in pack.items()}
            cols = [(pack[k], out[k]) for k in pack]
            n_kept = torch.empty(1, dtype=torch.int64, device=dev)
            sdf = torch.empty(n, device=dev)
            with torch.no_grad():
                t_op = ev_time(lambda: cabi.sdf_outlier_filter(ns, xyz, thr, cols, n_kept, ws, n=n), args.reps)
                t_sdf = ev_time(lambda: cabi.sdf_fwd(ns, xyz[:n], sdf), args.reps)
                kept = int(n_kept.item())
                pack_cpu = {k: v.cpu() for k, v in pack.items()}
                composition(net, pack_cpu, thr_double)  # warm-up
                ts, ts_sdf = [], []
                for _ in range(max(1, args.reps // 2)):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    ref, t_ref_sdf = composition(net, pack_cpu, thr_double)
                    ts.append(time.perf_counter() - t0)
                    ts_sdf.append(t_ref_sdf)
            same = ref["xyz"].shape[0] == kept and all(torch.equal(out[k][:kept].cpu().view(torch.int32), ref[k].view(torch.int32)) for k in pack)
            sel_ms = t_op - t_sdf
            row = 40
            bytes_sel = 4 * n + kept * row + kept * (row + 8)  # read the SDF and the kept rows, write the kept rows and their index
            print(json.dumps({"cloud": cloud, "N": N, "kept": kept, "thr": thr, "op_ms": round(t_op, 4), "op_sdf_ms": round(t_sdf, 4),
                              "op_select_gather_ms": round(sel_ms, 4), "select_gather_GBps": round(bytes_sel / (sel_ms * 1e-3) / 1e9, 1),
                              "select_gather_of_hbm_peak": round(bytes_sel / (sel_ms * 1e-3) / HBM, 3),
                              "composition_ms": round(1e3 * float(np.median(ts)), 2), "composition_sdf_ms": round(1e3 * float(np.median(ts_sdf)), 2),
                              "identical": bool(same)}), flush=True)
            del pack, out, cols, pack_cpu, ref, xyz, sdf
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
