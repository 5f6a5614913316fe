"""The joint stage driven the reference's way, for tests/test_gpu_gs_train.py and tools/gs_train_bench.py: `host_step(G, i)` runs iteration
i of a gstrain.GsTrainer with the operators GsTrainer.step uses, but in the reference's host-driven form (neural_mapping.cpp:396-523):
the sample std and the ray count read back with .item() and handed to the sampler and both SDF sites as host scalars, every logged value
read back with .item(), and sdf_train_callback's k_sample_std = max(mean(1 / isigma), bce_sigma) taken in torch from the forward's isigma
and written back. `snapshot(G)` / `restore(G, snap)` save and reset everything an iteration changes, so that one iteration can be run
both ways from the same state."""
import ctypes

import numpy as np
import torch

from gssdf_b200 import cabi
from gssdf_b200 import gstrain as GT

_f32 = np.float32


def host_step(G, i, log=True):
    T, S, rs = G.T, G.sdf, G.sdf.rs
    vm = G.load_frame(G.camera(i))
    T.normal_w = G.normal_w if GT.normal_on(i, G.refine_struct_start) else 0.0
    G.randns.normal_(generator=G.gen)
    S.draw()
    n_rays = int(S.n_rays_dev.item())          # k_batch_num
    delta = float(S.std_dev.item())            # k_sample_std
    n_live = torch.tensor([n_rays], dtype=torch.int32, device=G.dev)
    cabi.sdf_ray_batch(S.pack, S.rand, n_live, S.rays)
    rs.std = delta
    rs.sample(S.rays["origin"], S.rays["direction"], S.rays["depth"], S.rays["xyz"], n_live=n_live)  # host std
    dev_delta, T.delta_dev, T.delta = T.delta_dev, None, delta
    try:
        loss, sdf_loss = T.train_step(vm, G.Ks, G.gt, rs.xyz, rs.ray_sdf, G.randns, ray_n_live=rs.counts)
        # the isigma of the ray samples' forward (point_samples.pred_isigma), before the optimiser moves the net
        y1 = torch.empty(rs.cap, dtype=torch.float32, device=G.dev)
        cabi.sdf_fwd(T.sdf_net(), rs.xyz, torch.empty_like(y1), y1, n_variants=1, delta=delta, n_live=rs.counts)
        T.adam_clocks()
    finally:
        T.delta_dev = dev_delta
    if log:
        G.h_loss[i] = loss.item()
        G.h_sdf_loss[i] = sdf_loss.item()
        G.h_vis[i] = int(T.n_gate.item())
    pt_n = int(rs.counts[0].item())
    G.h_samples[i] = pt_n
    if pt_n > 0:
        inv = 1.0 / (1 + torch.nn.functional.softplus(y1[:pt_n], beta=100) * S.bce_isigma)
        m = float(_f32(float(inv.double().sum().item()) / pt_n))
        S.std_dev.fill_(m if not m < S.bce_sigma else S.bce_sigma)
    if G.outlier_remove and GT.outlier_due(i, G.outlier_interval):
        S.remove_outliers(i, total_iter=G.iters, net=T.sdf_net(), outlier_dist=G.outlier_dist)
    G.h_std[i:i + 1].copy_(S.std_dev)
    if GT.callback_due(i, G.iters):
        T.R.sh_degree = G.D.train_callback(i, G.iters)
    G.n_live_log.append(T.N_live)
    G.done = i + 1


def _struct_bytes(s):
    return ctypes.string_at(ctypes.addressof(s), ctypes.sizeof(s))


def snapshot(G):
    T, S, D = G.T, G.sdf, G.D
    c = lambda t: t.clone()
    return dict(
        T=dict(params=c(T._params), m=c(T._exp_avg), v=c(T._exp_avg_sq), anchors=c(T.anchors_buf), grad=c(T.flat_grad), half=c(T.table_half),
               packed=c(T.mlp_packed), sh_last=c(T.sh_last), replay=_struct_bytes(T.sh_replay.s), clocks=(T.t_splat, T.t_sh, T.t_sdf),
               lr=list(T.lr), sdf_lr=T.sdf_lr, N_live=T.N_live, stale=T._sh_stale, sh_degree=T.R.sh_degree, normal_w=T.normal_w,
               v_normals_dirty=getattr(T.R, "_v_normals_dirty", False), v_out_normals=c(T.R.v_out_normals)),
        S=dict(adapt=c(S.adapt), pack={k: c(v) for k, v in S._pack.items()}, N=S.N, gen=S.gen.get_state(), overflow=c(S.overflow)),
        D=dict(state={k: c(v) for k, v in D.state.items()}, gen=D.gen.get_state(), log=list(D.log)),
        G=dict(perm=None if G.perm is None else list(G.perm), cpu_gen=G.cpu_gen.get_state(), gen=G.gen.get_state(), n_live_log=list(G.n_live_log),
               done=G.done, h=[c(t) for t in (G.h_loss, G.h_sdf_loss, G.h_std, G.h_samples, G.h_vis)]))


def restore(G, snap):
    T, S, D = G.T, G.sdf, G.D
    t, s, d, g = snap["T"], snap["S"], snap["D"], snap["G"]
    T._params, T._exp_avg, T._exp_avg_sq, T.anchors_buf = t["params"].clone(), t["m"].clone(), t["v"].clone(), t["anchors"].clone()
    T.flat_grad.copy_(t["grad"]); T.table_half.copy_(t["half"]); T.mlp_packed.copy_(t["packed"]); T.sh_last.copy_(t["sh_last"])
    ctypes.memmove(ctypes.addressof(T.sh_replay.s), t["replay"], len(t["replay"]))
    T.t_splat, T.t_sh, T.t_sdf = t["clocks"]
    T.lr, T.sdf_lr, T._sh_stale, T.normal_w = list(t["lr"]), t["sdf_lr"], t["stale"], t["normal_w"]
    T.R.sh_degree = t["sh_degree"]
    T.R._v_normals_dirty = t["v_normals_dirty"]
    T.R.v_out_normals.copy_(t["v_out_normals"])
    T.N_live = t["N_live"]
    T.set_live(t["N_live"])  # rebinds the views (and the decoder struct) to the restored buffers
    S.adapt.copy_(s["adapt"])
    S._pack, S.N = {k: v.clone() for k, v in s["pack"].items()}, s["N"]
    S.gen.set_state(s["gen"]); S.overflow.copy_(s["overflow"])
    D.state = {k: v.clone() for k, v in d["state"].items()}
    D.gen.set_state(d["gen"]); D.log = list(d["log"])
    G.perm = None if g["perm"] is None else list(g["perm"])
    G.cpu_gen.set_state(g["cpu_gen"]); G.gen.set_state(g["gen"])
    G.n_live_log, G.done = list(g["n_live_log"]), g["done"]
    for dst, src in zip((G.h_loss, G.h_sdf_loss, G.h_std, G.h_samples, G.h_vis), g["h"]):
        dst.copy_(src)
