#!/usr/bin/env python
"""bench.py -- train-step/s (and Mrays/s) of the GS-SDF hot path on H100 (BASELINE.json metric).

A "step" is one pass of the hot path (SURVEY.md section 3.2 [A]-[D], rows a1-a12 + f-1 + the optimiser half of f-3 of section 8) over one
camera per rank: SDF stage on 32768 ray samples (hash grid + MLP, BCE + analytic eikonal + align with the tcnn double backward) ->
projection -> SH colour -> tile keys/sort/offsets -> rasterise -> post-ops -> GS<->SDF coupling on the visible splats' stochastic samples
(gated by visibility like the reference) -> photometric loss (0.8 L1 + 0.2 DSSIM) + depth L1 + normal-consistency + isotropic -> backward of
the render to {offsets, quaternion, scaling, opacity, SH} -> fused multi-tensor Adam over all 74 M parameters (zeroes the gradients,
refreshes the fp16 table shadow and the decoder's operand image). With N > 1 ranks (image-batch data parallel, replicated state) the flat
gradient is all-reduced over NCCL every step in two overlapped segments and every rank applies the same Adam update.

  value : whole-job steps/s with every input already resident in HBM (CUDA events, max over ranks)
  e2e   : the same through the public API with HOST buffers: per step the camera (viewmat, K) and the
          ground-truth image are copied from pinned host memory and the loss is read back (D2H)
  roofline     : dominant kernel (raster backward): algorithmic bytes (SURVEY 8d) on the intersections the launch PROCESSES / CUDA-event
                 time
  stock_cuda   : the reference fork's own CUDA kernels (oracle/_ref/gsplat_ref.so, compiled from /root/reference, test infrastructure) on
                 the same tensors on the same GPU, per stage, beside ours (SURVEY 8d / BASELINE.md 3.1-2) -- never part of the product path
  cpu_baseline : config c1 (256x256, 50 k splats, SH 0, MLP 2x32) run FOR REAL on the CPU oracle port incl. Adam (median step, SURVEY 8d),
                 next to the same c1 step on this GPU -- a measured ratio, nothing extrapolated

`--impl reference` times the reference's own CPU path: GS-SDF has none (every op CHECK_CUDAs, SURVEY 0.5), so this arm runs the oracle
port (oracle/, the CPU restatement of the reference kernels) with all host threads; each of its "steps" is a bounded SAMPLE of the
workload (1/4 linear resolution, 1/16 of the splats and ray samples) and `value` is the sample rate x 1/16 -- stated in config.workload.
"""
import argparse
import json
import math
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, os.path.join(ROOT, "gs-sdf_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402

WORKLOADS = {
    # name: (W, H, N splats, SH degree, isect capacity)
    "1080p-1M": (1920, 1080, 1_000_000, 3, 40_000_000),   # the config BASELINE.json's metric is quoted on (c4 per GPU)
    "c2": (1200, 680, 500_000, 3, 24_000_000),
    "c3": (1920, 1080, 2_000_000, 3, 60_000_000),
    "c5": (3840, 2160, 5_000_000, 3, 96_000_000),         # per GPU of the 8-GPU weak-scaling sweep
    "c1": (256, 256, 50_000, 0, 4_000_000),
    "tiny": (320, 192, 20_000, 3, 2_000_000),
}
# SDF sampling per workload: (rays per step, free samples per ray, surface samples per ray, capacity of the sample batch). Default: the
# reference's k_batch_pt_num = 32768 points from ~3277 rays with 3 free + 3 surface samples (config/base.yaml:21-23). c5 asks for 64 rays x
# 128 SDF samples per sampled pixel: 8192 rays x (124 free + 3 surface + voxel hits + the end point) ~ 1.07 M points per step.
SDF_SAMPLING = {"default": (3277, 3, 3, 49152), "c5": (8192, 124, 3, 1_310_720)}
CPU_SAMPLE_DIV = 4  # the CPU sample is the workload at 1/4 resolution per axis and 1/16 of the splats (1/16 of the work)


def peaks():
    try:
        return json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))), "measured"
    except Exception:
        return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0}, "H100 SXM data sheet"


class ClockSampler(threading.Thread):
    """SM clock / clock-event (throttle) reasons DURING the timed region, sampled in-process through NVML every 5 ms
    (nvidia-smi queries the same counters but takes ~100 ms per call); falls back to nvidia-smi when pynvml is unusable."""

    Q = "clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown," \
        "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"
    BITS = {"sw_power_cap": 0x4, "hw_slowdown": 0x8, "sw_thermal_slowdown": 0x20, "hw_thermal_slowdown": 0x40}

    def __init__(self, index, pci_bus_id=None):
        super().__init__(daemon=True)
        self.index, self.sm, self.reasons, self.max_mhz, self._stop_evt = index, [], set(), None, threading.Event()
        self.h = None
        try:
            import pynvml
            pynvml.nvmlInit()
            self.nv = pynvml
            self.h = pynvml.nvmlDeviceGetHandleByPciBusId(pci_bus_id.encode()) if pci_bus_id else pynvml.nvmlDeviceGetHandleByIndex(index)
            self.max_mhz = float(pynvml.nvmlDeviceGetMaxClockInfo(self.h, pynvml.NVML_CLOCK_SM))
        except Exception:
            self.h = None

    def _sample_nvml(self):
        nv = self.nv
        self.sm.append(float(nv.nvmlDeviceGetClockInfo(self.h, nv.NVML_CLOCK_SM)))
        get = getattr(nv, "nvmlDeviceGetCurrentClocksEventReasons", None) or nv.nvmlDeviceGetCurrentClocksThrottleReasons
        bits = int(get(self.h))
        self.reasons |= {n for n, b in self.BITS.items() if bits & b}

    def _sample_smi(self):
        out = subprocess.run(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-i", str(self.index)],
                             capture_output=True, text=True, timeout=5).stdout.strip()
        if out:
            r = [x.strip() for x in out.split(",")]
            self.sm.append(float(r[0]))
            self.max_mhz = max(self.max_mhz or 0.0, float(r[1]))
            self.reasons |= {n for n, v in zip(["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"], r[2:6])
                             if v.lower().startswith("active")}

    def run(self):
        while not self._stop_evt.is_set():
            try:
                self._sample_nvml() if self.h is not None else self._sample_smi()
            except Exception:
                pass
            self._stop_evt.wait(0.005 if self.h is not None else 0.2)

    def summary(self):
        self._stop_evt.set()
        return {"sm_mhz": float(np.median(self.sm)) if self.sm else None, "sm_max_mhz": self.max_mhz, "reasons": sorted(self.reasons),
                "samples": len(self.sm), "source": "nvml" if self.h is not None else "nvidia-smi"}


def pci_bus_id():
    """NVML-style bus id of the current CUDA device (robust to CUDA_VISIBLE_DEVICES remapping)."""
    try:
        import torch
        p = torch.cuda.get_device_properties(torch.cuda.current_device())
        return f"{p.pci_domain_id:08x}:{p.pci_bus_id:02x}:{p.pci_device_id:02x}.0"
    except Exception:
        return None


def cpu_dssim(x, y, w):
    """loss::dssim_loss on the host (numpy + scipy separable correlation, the reference's 11-tap window): w * (1 - mean SSIM) and d/dx."""
    from scipy.ndimage import correlate1d
    g = np.array([np.exp(-(np.floor((i - 11) / 2.0) ** 2) / 4.5) for i in range(11)], np.float32)
    g = (g / g.sum()).astype(np.float64)
    cv = lambda t, k: correlate1d(correlate1d(t, k, axis=0, mode="constant"), k, axis=1, mode="constant")
    x, y = x.astype(np.float64), y.astype(np.float64)
    mu1, mu2, s11, s22, s12 = cv(x, g), cv(y, g), cv(x * x, g), cv(y * y, g), cv(x * y, g)
    A1, A2 = 2 * mu1 * mu2 + 1e-4, 2 * (s12 - mu1 * mu2) + 9e-4
    B1, B2 = mu1 * mu1 + mu2 * mu2 + 1e-4, (s11 - mu1 * mu1) + (s22 - mu2 * mu2) + 9e-4
    S = A1 * A2 / (B1 * B2)
    dm = 2 * mu2 * (A2 - A1) / (B1 * B2) - S * (2 * mu1 / B1 - 2 * mu1 / B2)
    d11, d12 = -S / B2, 2 * A1 / (B1 * B2)
    gf = g[::-1].copy()
    grad = (cv(dm, gf) + 2 * x * cv(d11, gf) + y * cv(d12, gf)) * (-w / S.size)
    return w * (1 - S.mean()), grad.astype(np.float32)


def cpu_oracle_step(O, S, sc, V, K, W, H, deg, rn, gt):
    """One hot-path step on the CPU oracle port (fp32 restatement, OpenMP)."""
    p = O.project2dgs_fwd(sc["means"], sc["quats"], sc["scales"], V, K, W, H, S.NEAR, S.FAR, 0.0, rn, "f32")
    col, dirs = O.view_colors_fwd(V, sc["means"], p["radii"], sc["sh"], p["camera_ids"], p["gaussian_ids"], deg, "f32")
    tw, th = (W + 15) // 16, (H + 15) // 16
    _, ids, flat = O.isect_tiles(p["means2d"], p["radii"], p["depths"], p["camera_ids"], 1, 16, tw, th)
    off = O.isect_offsets(ids, 1, tw, th)
    op = sc["opacities"][p["gaussian_ids"]]
    r = O.raster2dgs_fwd(p["ray_transforms"], col, op, p["normals"], W, H, 16, off, flat, None, "f32")
    ed = np.nan_to_num(r["render_depths"] / r["render_alphas"])
    out = np.concatenate([r["render_colors"], ed], -1)
    d = out - gt
    npx = W * H
    # photometric loss of the step: 0.8 L1 + 0.2 (1 - SSIM) on rgb (config/base.yaml:35-36) + 0.1 L1 on the expected depth
    loss = 0.8 * np.abs(d[..., :3]).sum() / (3 * npx) + 0.1 * np.abs(d[..., 3:]).sum() / npx
    v_out = np.sign(d) * np.array([0.8 / (3 * npx)] * 3 + [0.1 / npx], np.float32)
    for ch in range(3):
        l_s, g_s = cpu_dssim(out[0, :, :, ch], gt[0, :, :, ch], 0.2 / 3)
        loss += l_s
        v_out[0, :, :, ch] += g_s
    fin = np.isfinite(r["render_depths"] / np.where(r["render_alphas"] == 0, np.nan, r["render_alphas"]))
    v_dep = np.where(fin, v_out[..., 3:] / np.where(fin, r["render_alphas"], 1), 0).astype(np.float32)
    v_alp = np.where(fin, -v_out[..., 3:] * r["render_depths"] / np.where(fin, r["render_alphas"], 1) ** 2, 0).astype(np.float32)
    z3 = np.zeros((1, H, W, 3), np.float32)
    rb = O.raster2dgs_bwd(p["ray_transforms"], col, op, p["normals"], W, H, 16, off, flat, r["render_alphas"], r["render_Ts"],
                          r["last_ids"], r["median_ids"], np.ascontiguousarray(v_out[..., :3]), v_dep, v_alp, z3,
                          np.zeros((1, H, W, 1), np.float32), None, None, "f32")
    vcm = rb["v_colors"] * (col > 0)
    O.sh_bwd(deg, dirs, sc["sh"][p["gaussian_ids"]], vcm, None, "f32")
    O.project2dgs_bwd(sc["means"], sc["quats"], sc["scales"], V, K, p["camera_ids"], p["gaussian_ids"], p["ray_transforms"],
                      p["randns"], rb["v_means2d"], np.zeros(p["nnz"], np.float32), rb["v_ray_transforms"], rb["v_normals"],
                      np.zeros((p["nnz"], 3), np.float32), "f32")
    return float(loss), p["nnz"], len(flat), p, r


def cpu_oracle_sdf(O, pts, table, mlp, hidden, n_hidden, gt=None, weights=None, delta=0.1, analytic=True, align_w=0.1):
    """SDF stage on the oracle port: 7 evaluations per point, losses, backward (table + decoder + d/dx of the base point).
    analytic: eikonal + align on the analytic gradient with its double backward (reference default), else the 6-offset eikonal."""
    n = len(pts)
    offs = np.array([[0, 0, 0], [1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.float32) * np.float32(delta)
    x01 = (((pts[None] + offs[:, None]).reshape(-1, 3)).astype(np.float32) * np.float32(1.0 / 14.0) + np.float32(0.5)).astype(np.float32)
    sdf, y1, _ = O.sdf_fwd(x01, table, mlp, hidden, n_hidden)
    if not analytic:
        loss, vs, vy = O.sdf_losses(sdf, y1, n, 7, gt, weights, 10.0, 1.0 if gt is not None else 0.0, 0.1, 1e-3, delta)
        O.sdf_bwd(x01, table, mlp, vs, vy, hidden, n_hidden)
        return loss
    loss, vs, vy = O.sdf_losses(sdf, y1, n, 7, gt, weights, 10.0, 1.0 if gt is not None else 0.0, 0.0, 1e-3, delta)
    vs, vy = np.asarray(vs).reshape(7, n)[0].astype(np.float32), np.asarray(vy).reshape(7, n)[0].astype(np.float32)
    O.sdf_bwd(x01[:n], table, mlp, vs, vy, hidden, n_hidden)  # first order: only the base evaluations carry cotangents
    g = O.sdf_grad_analytic(x01[:n], table, mlp, hidden, n_hidden).astype(np.float64) / 14.0  # world units
    s7 = np.asarray(sdf, np.float64).reshape(7, n)
    gnum = np.stack([s7[1] - s7[2], s7[3] - s7[4], s7[5] - s7[6]], 1) * (0.5 / delta)
    nrm = np.maximum(np.linalg.norm(g, axis=1), 1e-30)
    loss += 0.1 * np.mean((nrm - 1) ** 2) + align_w * np.mean(np.abs(g - gnum))
    c = (0.1 / n) * (2 * (nrm - 1) / nrm)[:, None] * g + (align_w / (3 * n)) * np.sign(g - gnum)
    O.sdf_grad_analytic_bwd(x01[:n], table, mlp, (c / 14.0).astype(np.float32), hidden, n_hidden)
    return loss


class CpuAdam:
    """torch::optim::Adam (eps 1e-15) on numpy arrays, for the CPU arms (the reference's step ends with Adam.step())."""

    def __init__(self, params, lrs):
        self.p, self.lr, self.t = params, lrs, 0
        self.m = [np.zeros_like(x) for x in params]
        self.v = [np.zeros_like(x) for x in params]

    def step(self, grads):
        self.t += 1
        bc1, bc2 = 1 - 0.9 ** self.t, 1 - 0.999 ** self.t
        for p_, g, m, v, lr in zip(self.p, grads, self.m, self.v, self.lr):
            g = g.astype(np.float32, copy=False).reshape(p_.shape)
            m *= 0.9
            m += 0.1 * g
            v *= 0.999
            v += 0.001 * g * g
            p_ -= (lr / bc1) * (m / (np.sqrt(v) / math.sqrt(bc2) + 1e-15))


def cpu_full_step(O, S, sc, V, K, W, H, deg, rn, gt, table, mlp, hidden, n_hidden, ray, ray_gt, adam=None, analytic=True):
    """[A]-[D] (+ Adam) on the oracle port; gradients w.r.t. the ACTIVATED splat parameters (the activations' chain rule is a handful of
    elementwise numpy ops, negligible next to the render)."""
    cpu_oracle_sdf(O, ray, table, mlp, hidden, n_hidden, gt=ray_gt, analytic=analytic)
    loss, nnz, I, p, r = cpu_oracle_step(O, S, sc, V, K, W, H, deg, rn, gt)
    vis = np.asarray(r["visibilities"], np.float32)[:, 0]
    sel = vis > 0.1  # the reference's sample gate (neural_mapping.cpp:428-437)
    w = (p["sample_weights"][:, 0] * vis).astype(np.float32)
    if sel.any():
        cpu_oracle_sdf(O, p["samples"][sel], table, mlp, hidden, n_hidden, weights=w[sel], analytic=analytic)
    if adam is not None:  # dense update of every parameter tensor with stand-in gradients of the right size (the oracle calls above
        adam.step(adam.grads)  # produce them; they are not threaded through to keep the oracle API unchanged)
    return loss, nnz, I


def run_cpu_c1(budget_s=20.0, max_steps=20, warmup=3):
    """SURVEY 8d: the CPU baseline is config c1 (256x256, 50 k splats, SH degree 0, MLP 2x32), the full step incl. Adam, for real."""
    from gssdf_b200 import scene as S
    from oracle import oracle as O
    O.build()
    W, H, N, deg, _ = WORKLOADS["c1"]
    sc = S.box_scene(N, deg, seed=0)
    V, K = S.cameras([0], W, H)
    rn = S.randns(N)
    gt = np.random.default_rng(3).random((1, H, W, 4), dtype=np.float32)
    cores = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    os.environ["OMP_NUM_THREADS"] = str(cores)
    O.set_threads(cores)
    try:
        import threadpoolctl
        threadpoolctl.threadpool_limits(limits=cores)
    except Exception:
        pass
    rng = np.random.default_rng(5)
    n_table, _ = O.grid_setup()
    table = rng.uniform(-1e-4, 1e-4, n_table).astype(np.float32)
    hidden, n_hidden = 32, 1
    dims = [32] + [hidden] * (1 + n_hidden) + [2]
    mlp = np.concatenate([np.concatenate([rng.uniform(-1, 1, o * k) / np.sqrt(k), rng.uniform(-1, 1, o) / np.sqrt(k)])
                          for k, o in zip(dims[:-1], dims[1:])]).astype(np.float32)
    # sample generation like the GPU arm: occupancy octree of the scene (level 8 over 14 m), 3277 depth rays per step through the
    # kaolin-style level-by-level ray trace + NeuralSLAM::sample (oracle/octree_oracle.c, oracle.sdf_sample_generation)
    n_rays, level, leaf = 3277, 8, 14.0 / 256
    tree = O.octree_from_points(O.quantize_points(sc["means"] * np.float32(2.0 / 14.0), level), level)
    ro = ((rng.uniform(0, 1, (1 << 16, 3)) - 0.5) * S.BOX).astype(np.float32)
    rend = sc["means"][rng.integers(0, N, 1 << 16)]
    rdep = np.linalg.norm(rend - ro, axis=1).astype(np.float32)
    rdir = ((rend - ro) / rdep[:, None]).astype(np.float32)
    params = [sc["means"], sc["quats"], sc["scales"], sc["opacities"], sc["sh"], table, mlp]
    adam = CpuAdam(params, [1.6e-4, 1e-3, 5e-3, 5e-2, 2.5e-3, 5e-3, 5e-3])
    adam.grads = [np.full_like(x, 1e-9) for x in params]
    ts, nnz, I, n_ray = [], 0, 0, 0
    t_all = time.perf_counter()
    for i in range(warmup + max_steps):
        t0 = time.perf_counter()
        k = (i * n_rays) % ((1 << 16) - n_rays)
        smp, _ = O.sdf_sample_generation(tree, ro[k:k + n_rays], rdir[k:k + n_rays], rdep[k:k + n_rays], rend[k:k + n_rays], np.zeros(3), 14.0,
                                         rng.uniform(0, 1, 64 * n_rays), rng.uniform(0, 1, (n_rays, 3)), rng.standard_normal((n_rays, 3)), 3, 3,
                                         0.1, 3 * leaf, [-7.0] * 3, [7.0] * 3)
        ray, ray_gt, n_ray = smp["xyz"], smp["ray_sdf"][:, 0].copy(), len(smp["xyz"])
        # numerical (6-offset) eikonal like the GPU arm at c1: the fused analytic kernel covers the 3x64 decoder only
        _, nnz, I = cpu_full_step(O, S, sc, V, K, W, H, deg, rn, gt, table, mlp, hidden, n_hidden, ray, ray_gt, adam, analytic=False)
        if i >= warmup:
            ts.append(time.perf_counter() - t0)
        if time.perf_counter() - t_all > budget_s and len(ts) >= 3:
            break
    med = float(np.median(ts))
    return dict(value=1.0 / med, unit="step/s", cores=cores, kind="port", config="c1",
                sample=f"config c1 run for real, nothing scaled: {W}x{H}, {N} splats, SH deg {deg}, MLP 2x32, octree sample generation of {n_rays} rays -> {n_ray} ray samples + {nnz} "
                       f"splat samples x7 SDF evaluations, numerical eikonal (as the GPU arm at c1), L1 + DSSIM, Adam over {sum(x.size for x in params)} "
                       f"parameters; median of {len(ts)} steps after {warmup} warm-ups = {med * 1e3:.0f} ms (nnz={nnz}, n_isects={I}); "
                       f"C + OpenMP fp32 oracle port, numpy/scipy glue")


def run_cpu_sample(workload, steps, warmup, budget_s=25.0):
    """Times the oracle port on a bounded sample: the workload at 1/4 linear resolution with 1/16 of the splats
    (same screen coverage per splat, 1/16 of every unit count); returns full-workload-equivalent steps/s."""
    from gssdf_b200 import scene as S
    from oracle import oracle as O
    O.build()
    W, H, N, deg, _ = WORKLOADS[workload]
    Ws, Hs, Ns = max(W // CPU_SAMPLE_DIV, 16), max(H // CPU_SAMPLE_DIV, 16), max(N // CPU_SAMPLE_DIV ** 2, 64)
    # 1/16 of the splats, each 4x larger in world space: same pixel footprint per splat at 1/4 resolution, hence the
    # same per-tile depth complexity as the full workload and 1/16 of its nnz, n_isects, tiles and pixels
    sc = S.box_scene(Ns, deg, seed=0, scale_mult=math.sqrt(1.0e6 / N) * CPU_SAMPLE_DIV)
    V, K = S.cameras([0], Ws, Hs)
    rn = S.randns(Ns)
    gt = np.random.default_rng(3).random((1, Hs, Ws, 4), dtype=np.float32)
    cores = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    os.environ["OMP_NUM_THREADS"] = str(cores)  # torchrun exports OMP_NUM_THREADS=1 into its ranks: the CPU arm uses every host core
    O.set_threads(cores)
    try:  # numpy's BLAS pool read OMP_NUM_THREADS=1 at import time under torchrun
        import threadpoolctl
        threadpoolctl.threadpool_limits(limits=cores)
    except Exception:
        pass
    rng = np.random.default_rng(5)
    n_table, _ = O.grid_setup()
    table = rng.uniform(-1e-4, 1e-4, n_table).astype(np.float32)
    hidden, n_hidden = (32, 1) if workload == "c1" else (64, 3)
    dims = [32] + [hidden] * (1 + n_hidden) + [2]
    mlp = np.concatenate([np.concatenate([rng.uniform(-1, 1, o * k) / np.sqrt(k), rng.uniform(-1, 1, o) / np.sqrt(k)])
                          for k, o in zip(dims[:-1], dims[1:])]).astype(np.float32)
    n_ray = 32768 // CPU_SAMPLE_DIV ** 2
    ray = (rng.uniform(-1, 1, (n_ray, 3)) * (S.BOX + 0.3)).astype(np.float32)
    ray_gt = np.clip((S.BOX - np.abs(ray)).min(1), -0.3, 0.3).astype(np.float32)

    params = [sc["means"], sc["quats"], sc["scales"], sc["opacities"], sc["sh"], table, mlp]
    adam = CpuAdam(params, [1.6e-4, 1e-3, 5e-3, 5e-2, 2.5e-3, 5e-3, 5e-3])
    adam.grads = [np.full_like(x, 1e-9) for x in params]

    def full_step():
        return cpu_full_step(O, S, sc, V, K, Ws, Hs, deg, rn, gt, table, mlp, hidden, n_hidden, ray, ray_gt, adam)

    for _ in range(max(1, min(warmup, 2))):
        full_step()
    t0 = time.perf_counter()
    ts = []
    for _ in range(max(steps, 1)):
        t1 = time.perf_counter()
        _, nnz, I = full_step()
        ts.append(time.perf_counter() - t1)
        if time.perf_counter() - t0 > budget_s:
            break
    dt, done = float(np.median(ts)), len(ts)
    frac = (Ws * Hs) / float(W * H)
    value = (1.0 / dt) * frac  # sample steps/s scaled by the work fraction = full-workload-equivalent steps/s
    return dict(value=value, unit="step/s", cores=cores, kind="port", sample_steps_per_s=1.0 / dt, sample_fraction=frac,
                sample=f"median of {done} oracle steps (C, OpenMP, fp32, incl. numpy Adam over the full 15.3 M-entry table) of a BOUNDED SAMPLE "
                       f"of the workload: 1/{CPU_SAMPLE_DIV} linear resolution ({Ws}x{Hs}), {Ns} splats, nnz={nnz}, n_isects={I}, "
                       f"{n_ray}+gated splat samples x7 SDF evaluations, analytic eikonal + align with double backward: {dt * 1e3:.0f} ms "
                       f"each; value = sample steps/s x {frac:.4f} (an extrapolation by work fraction, see cpu_baseline for a measured "
                       f"like-for-like c1 pair)"), W, H


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--workload", default="1080p-1M", choices=sorted(WORKLOADS))
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--eikonal", default="analytic", choices=["analytic", "numerical"],
                    help="analytic: eikonal + align on d sdf/dx with double backward (reference default); numerical: 6-offset gradient")
    ap.add_argument("--same-cameras", action="store_true", help="N>1: every rank renders the same camera pose at every step (no load imbalance); "
                    "default: one shared pool of poses, rank r a fixed number of poses ahead in the cycle")
    ap.add_argument("--no-stock-cuda", action="store_true", help="skip the reference-fork CUDA leg (oracle/_ref/gsplat_ref.so)")
    ap.add_argument("--overlap", type=int, default=1, choices=[0, 1, 2, 3],
                    help="schedule of the SDF-only work (sample generation, [A], [C]): 0 = in line on one stream, 1 = on a second stream beside the "
                         "render (equal priority), 2 = second stream at high priority, 3 = render stream at high priority")
    ap.add_argument("--no-cover", action="store_true", help="A/B (N > 1, two-stream schedule): keep sample generation + [A] on the second stream "
                    "even while a dense all-reduce is in flight")
    ap.add_argument("--dense-allreduce", action="store_true", help="A/B (N > 1): always all-reduce the dense splat segment (no sparse row exchange)")
    ap.add_argument("--nccl-high-priority", action="store_true", help="A/B (N > 1): run NCCL's kernels on a high-priority stream")
    ap.add_argument("--dump-outputs", metavar="DIR", help="after the timed steps, write what the last timed step computed (losses, "
                    "rendered image and normals, updated parameters) as DIR/<name>.npy; arrays too large for the 64 MB total are fixed, "
                    "seeded samples of their elements")
    ap.add_argument("--l2-persist", action="store_true", help="A/B: pin the fp16 hash-table shadow in L2 (gssdf_l2_persist); measured: no effect")
    args = ap.parse_args()
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    W, H, N, deg, isect_cap = WORKLOADS[args.workload]
    cfg = {"workload": f"{args.workload}: {W}x{H}, {N} splats, SH deg {deg}, synthetic box scene seed 0 (SURVEY 8d), tile 16, packed, "
                       f"1 camera/rank/step", "timing": "CUDA events; inputs (232 B/splat state + images) exceed the 50 MB L2, no flush",
           "parallelism": (f"image-parallel dp{world}, replicated state, one pool of 8 camera poses, rank r renders pose (step + r * {max(8 // world, 1)}) mod 8"
                           f"{' (--same-cameras: the same pose on every rank)' if args.same_cameras else ''}, 2 NCCL exchanges/step: SDF segment (all-reduce) under "
                           f"the render backward; splat segment after the backward, as an all-gather of the ranks' visible rows when they are "
                           f"less than half the dense segment, else a dense all-reduce{' (--dense-allreduce: always dense)' if args.dense_allreduce else ''}; replicated Adam "
                           f"with grad_scale 1/{world}")
           if world > 1 else "single GPU",
           "schedule": ["one stream, stages in line", "SDF-only work (sample generation, [A], [C]) on a second stream beside the render",
                        "SDF-only work on a second, high-priority stream", "render on a high-priority stream, SDF-only work on a second stream"][args.overlap]}

    if args.impl == "reference":
        if rank != 0:
            return 0
        cb, _, _ = run_cpu_sample(args.workload, max(args.steps, 1), args.warmup)
        cfg = dict(cfg, workload=cfg["workload"] + f"; THIS ARM: each step is a bounded sample of that workload at 1/{CPU_SAMPLE_DIV} linear "
                   f"resolution with 1/{CPU_SAMPLE_DIV ** 2} of the splats and ray samples, value = measured sample steps/s "
                   f"({cb['sample_steps_per_s']:.4f}) x {cb['sample_fraction']:.4f}", parallelism=f"{cb['cores']} host threads (OpenMP)")
        line = {"impl": "reference", "metric": "train_steps_per_s", "value": cb["value"], "unit": "step/s", "n_gpus": args.gpus,
                "steps": args.steps, "warmup": args.warmup, "ms_per_step": 1e3 / cb["value"], "higher_is_better": True,
                "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic", "config": cfg, "cpu_baseline": cb,
                "e2e": {"value": cb["value"], "unit": "step/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
                "mrays_per_s": cb["value"] * W * H / 1e6,
                "note": "GS-SDF has no CPU implementation of this path (SURVEY 0.5); this arm is the oracle port of the reference kernels"}
        print(json.dumps(line))
        return 0

    import torch
    import torch.distributed as dist

    from gssdf_b200 import render
    from gssdf_b200 import scene as S
    assert torch.cuda.is_available(), "bench.py needs a CUDA device (no CPU fallback exists)"
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        opts = None
        if args.nccl_high_priority:  # NCCL's kernels on a high-priority stream: their CTAs are placed as soon as any CTA slot frees up
            opts = dist.ProcessGroupNCCL.Options(is_high_priority_stream=True)
        dist.init_process_group("nccl", device_id=dev, pg_options=opts)

    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)

    def build_trainer(workload, eikonal):
        """Trainer + its replicated state for one workload: synthetic box scene (SURVEY 8d) as RAW NeuralGS parameters (anchors = centres,
        offsets = 0, scaling = log s, opacity = logit(o), features_dc | features_rest), tcnn-initialised table, torch-initialised decoder."""
        W, H, N, deg, isect_cap = WORKLOADS[workload]
        sc_np = S.box_scene(N, deg, seed=0)
        sc_act = {k: t(v) for k, v in sc_np.items()}
        K_sh = (deg + 1) ** 2
        sdf_cfg = dict(n_levels=16, n_features=2, log2_hashmap_size=19, base_resolution=32, per_level_scale=2.0,
                       hidden_dim=32 if workload == "c1" else 64, n_hidden=1 if workload == "c1" else 3)
        T = render.GsSdfTrainer(N, K_sh, W, H, dev, isect_cap, sdf_cfg, n_ray_samples=SDF_SAMPLING.get(workload, SDF_SAMPLING["default"])[3],
                                sh_degree=deg, origin=(0.0, 0.0, 0.0),
                                map_size=14.0, eikonal_mode=(1 if eikonal == "analytic" and sdf_cfg["hidden_dim"] == 64 else 0),
                                normal_weight=0.01, isotropic_weight=0.05)  # config/base.yaml:43-46
        T.l2_persist = args.l2_persist
        T.overlap = args.overlap > 0 and T.mlp_mode == 1
        T.sdf_stream_priority = -1 if args.overlap == 2 else 0
        gen = torch.Generator(dev).manual_seed(5)  # replicated parameters: same on every rank
        table = (torch.rand(T.n_table, device=dev, generator=gen) * 2 - 1) * 1e-4  # tcnn grid init U(+-1e-4) (grid.h:1059-1062)
        chunks, dims = [], [32] + [sdf_cfg["hidden_dim"]] * (1 + sdf_cfg["n_hidden"]) + [2]
        for k_, o_ in zip(dims[:-1], dims[1:]):  # torch::nn::Linear default init
            b_ = 1.0 / math.sqrt(k_)
            chunks += [(torch.rand(o_ * k_, device=dev, generator=gen) * 2 - 1) * b_, (torch.rand(o_, device=dev, generator=gen) * 2 - 1) * b_]
        op_ = np.clip(sc_np["opacities"], 1e-6, 1 - 1e-6)
        T.load(sc_act["means"], torch.zeros(N, 3, device=dev), sc_act["quats"], t(np.log(sc_np["scales"]).astype(np.float32)),
               t(np.log(op_ / (1 - op_)).astype(np.float32)), t(sc_np["sh"][:, :1].copy()),
               t(sc_np["sh"][:, 1:].copy()) if deg > 0 else None, table, torch.cat(chunks))
        return T, sc_act, (W, H, N, deg)

    # SDF ray samples (rows a13 / f-2): k_batch_num depth rays per step go through the octree ray-march + free / surface sampling of
    # NeuralSLAM::sample; the reference adapts k_batch_num so that the batch holds ~k_batch_pt_num = 32768 points (neural_mapping.cpp:324-330)
    # -- ~10 points per ray here. n_ray = capacity of the sample batch the SDF stage is sized for.
    OCT_LEVEL, LEAF = 8, 14.0 / 256
    N_RAYS, N_FREE, N_SURF, n_ray = SDF_SAMPLING.get(args.workload, SDF_SAMPLING["default"])
    from gssdf_b200 import octree as OT
    box = torch.tensor(S.BOX, device=dev, dtype=torch.float32)

    class Sampling:
        """occupancy octree of the scene (leaf 5.5 cm, SubMap of 14 m like the SDF grid) + a device-resident pack of depth rays (sensor
        positions inside the room looking at wall points: the stand-in for the dataset's train_depth_pack_) + the RaySampler"""

        def __init__(self, T_, means, seed):
            self.tree = OT.OctreeAS.from_quantized_points(OT.quantize_points(means * (2.0 / 14.0), OCT_LEVEL), OCT_LEVEL, dev,
                                                          origin=(0.0, 0.0, 0.0), map_size=14.0)
            g_ = torch.Generator(dev).manual_seed(seed)
            self.n_pack = 1 << 18
            self.o = ((torch.rand(self.n_pack, 3, device=dev, generator=g_) - 0.5) * box).contiguous()
            self.end = means[torch.randint(0, means.shape[0], (self.n_pack,), device=dev, generator=g_)].contiguous()
            self.depth = (self.end - self.o).norm(dim=1).contiguous()
            self.dir = ((self.end - self.o) / self.depth[:, None]).contiguous()
            nr_, nf_, ns_, cap_ = (N_RAYS, N_FREE, N_SURF, n_ray) if T_.n_ray == n_ray else SDF_SAMPLING["default"]
            self.n_rays = nr_
            self.rs = OT.RaySampler(self.tree, nr_, dev, 1, nf_, ns_, sample_std=T_.delta, truncated_dis=3 * LEAF, xyz_min=(-7.0,) * 3,
                                    xyz_max=(7.0,) * 3, nugget_cap=16 * nr_, cap=cap_)
            T_.set_octree(self.tree)

        def draw(self, i):
            nr_ = self.n_rays
            k = (i * nr_) % (self.n_pack - nr_)  # the reference indexes torch::rand rays of the pack (neural_mapping.cpp:145-156)
            self.rs.draw()
            self.rs.sample(self.o[k:k + nr_], self.dir[k:k + nr_], self.depth[k:k + nr_], self.end[k:k + nr_])
            return self.rs.xyz, self.rs.ray_sdf, self.rs.counts

    if args.overlap == 3:  # everything below is enqueued on a high-priority stream; the SDF stream keeps the default priority
        torch.cuda.set_stream(torch.cuda.Stream(device=dev, priority=-1))
    T, sc_act, _ = build_trainer(args.workload, args.eikonal)
    R = T.R
    K_sh = (deg + 1) ** 2
    SP = Sampling(T, sc_act["means"], 50 + rank)  # each rank draws its own rays
    n_cams = 8
    # image-batch data parallelism = "per-frame render on each rank" (north_star): every rank draws from the SAME pool of camera poses
    # (like ranks sharing one dataset), rank r being cam_shift poses ahead in the cycle -- at every step the ranks render different poses,
    # so the per-step load imbalance of real training is part of the measurement, while the work per rank averaged over the cycle is the
    # same for every rank and every N (weak scaling). --same-cameras: identical pose at every step on every rank (no imbalance).
    cam_shift = 0 if (args.same_cameras or world == 1) else rank * max(n_cams // world, 1)
    cam_of = lambda i: (i + cam_shift) % n_cams
    cams = [S.camera(i, W, H) for i in range(n_cams)]
    torch.manual_seed(1234 + rank)  # randns stream

    def gt_images(Tr, act, cam_list, Wc, Hc):
        """ground truth: the same scene rendered with perturbed colours (SURVEY 8d), produced once on the device"""
        sh_gt = act["sh"] + 0.1 * torch.randn(act["sh"].shape, device=dev, generator=torch.Generator(dev).manual_seed(3))
        out = []
        for V_, K_ in cam_list:
            Tr.R.forward(act["means"], act["quats"], act["scales"], act["opacities"], sh_gt, t(V_[None]), t(K_[None]))
            out.append(Tr.R.out_colors.clone())
        return out

    gts = gt_images(T, sc_act, cams, W, H)
    randn_buf = torch.empty(N, 2, device=dev)
    torch.cuda.synchronize()
    dev_cams = [(t(V[None]), t(Kc[None])) for V, Kc in cams]
    host_cams = [(torch.from_numpy(V[None].copy()).pin_memory(), torch.from_numpy(Kc[None].copy()).pin_memory()) for V, Kc in cams]
    host_gts = [g.cpu().pin_memory() for g in gts]
    loss_host = torch.empty(1).pin_memory()

    n_splat_grad = R.flat_grad.numel()
    # Data-parallel gradient exchange (gssdf_b200/parallel.py:GradientExchange): two NCCL all-reduces per step, both overlapped with
    # compute that does not depend on them -- the hash-table + decoder segment (61 MB) under the render backward [D] of the same step,
    # the splat segment (236 MB) under stage [A] of the NEXT step. Each segment's Adam update (grad_scale = 1 / world) runs as soon as its
    # reduction is complete: SDF groups right after the step, splat groups just before the next render touches the splats.
    from gssdf_b200 import densify, parallel
    # gssdf_b200/parallel.py: the step + its two overlapped exchanges + per-segment Adam (splat segment: visible rows when that is smaller)
    DP = parallel.DataParallelStep(T, world, sparse_rows=not args.dense_allreduce)
    DP.cover_dense_exchange = not args.no_cover
    DEN = densify.Densifier(T, num_train_data=n_cams, sh_degree=deg)

    def pre_render():
        DP.flush()

    def step_resident(i):
        V, Kc = dev_cams[cam_of(i)]
        R._mark("step_begin")
        randn_buf.normal_()  # the reference draws randns on the device every render (Projection.cpp:728)
        with T.sdf_stage():
            ray_xyz, ray_gt, ray_cnt = SP.draw(i)
        loss, sdf_loss = DP.step(V, Kc, gts[cam_of(i)], ray_xyz, ray_gt, randn_buf, ray_n_live=ray_cnt)
        DEN.update_state()  # NeuralGS::update_state: per-iteration densification statistics (the every-100-iterations surgery is not timed)
        R._mark("densify_stats")
        return loss, sdf_loss

    # end-to-end path: every step's inputs (camera pose, intrinsics, ground-truth image) come from pinned HOST memory and the loss is
    # read back to the host every step. The copy of step i+1's inputs is enqueued on a copy stream while step i computes (two device
    # input slots), like a training loop with a prefetching data loader; every copy still happens inside the timed region.
    copy_stream = torch.cuda.Stream(device=dev)
    slots = [dict(V=torch.empty(1, 4, 4, device=dev), K=torch.empty(1, 3, 3, device=dev), gt=torch.empty(1, H, W, 4, device=dev),
                  ready=torch.cuda.Event(), free=torch.cuda.Event()) for _ in range(2)]

    def prefetch(i):
        sl = slots[i % 2]
        with torch.cuda.stream(copy_stream):
            copy_stream.wait_event(sl["free"])  # the step that last used this slot has finished with it
            hv, hk = host_cams[cam_of(i)]
            sl["V"].copy_(hv, non_blocking=True)
            sl["K"].copy_(hk, non_blocking=True)
            sl["gt"].copy_(host_gts[cam_of(i)], non_blocking=True)
            sl["ready"].record(copy_stream)

    def step_e2e(i, last=False):
        if i == 0:
            prefetch(0)
        if not last:
            prefetch(i + 1)
        sl = slots[i % 2]
        cur = torch.cuda.current_stream()
        cur.wait_event(sl["ready"])
        randn_buf.normal_()
        with T.sdf_stage():
            ray_xyz, ray_gt, ray_cnt = SP.draw(i)
        loss, _sdf_loss = DP.step(sl["V"], sl["K"], sl["gt"], ray_xyz, ray_gt, randn_buf, ray_n_live=ray_cnt)
        sl["free"].record(cur)
        DEN.update_state()
        loss_host.copy_(loss, non_blocking=True)
        cur.synchronize()  # the caller reads the loss every step (neural_mapping.cpp:505-514)
        return float(loss_host[0])

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(fn, steps, sampler=None):
        barrier()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        if sampler:
            sampler.start()
        ev0.record()
        for i in range(steps):
            fn(i)
        if world > 1:
            pre_render()  # the last step's splat all-reduce and splat Adam belong to the timed region
        ev1.record()
        barrier()
        ms = ev0.elapsed_time(ev1)
        if world > 1:
            tm = torch.tensor([ms], device=dev)
            dist.all_reduce(tm, op=dist.ReduceOp.MAX)
            ms = float(tm[0])
        return ms

    for i in range(max(args.warmup, 3)):
        step_resident(i)
    if world > 1:
        pre_render()
    cnt = R.read_counts()
    assert not cnt["nnz_overflow"] and not cnt["isect_overflow"], f"capacity overflow: {cnt}"
    # the timed region; the library records one CUDA-event pair per step around each raster kernel
    mk = lambda: (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
    prof_f, prof_b = [mk() for _ in range(args.steps)], [mk() for _ in range(args.steps)]
    for e0, e1 in prof_f + prof_b:
        e0.record(); e1.record()  # creates the cudaEvent_t handles
    torch.cuda.synchronize()
    sampler = ClockSampler(local, pci_bus_id()) if rank == 0 else None

    last_out = {}

    def step_prof(i):
        R.prof_fwd, R.prof_bwd = prof_f[i], prof_b[i]
        last_out["loss"], last_out["sdf_loss"] = step_resident(i)

    ms_total = timed(step_prof, args.steps, sampler)
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, dict(last_out, render_colors=R.out_colors, render_normals=R.out_normals, params=T.params))
    fwd_ms = [a.elapsed_time(b) for a, b in prof_f]
    bwd_ms = [a.elapsed_time(b) for a, b in prof_b]
    R.prof_fwd = R.prof_bwd = None
    clocks = sampler.summary() if sampler else None
    ms_step = ms_total / args.steps
    value = world * 1e3 / ms_step  # images (train steps of one camera) per second over the whole job
    last_loss = float(T.R.loss[0])
    cnt_end = R.read_counts()
    sdf_counts = {"ray_samples": int(SP.rs.counts[0]), "ray_voxel_hits": int(SP.rs.counts[1]), "sample_overflow": int(SP.rs.counts[2]),
                  "rays": N_RAYS, "splat_samples_gated": int(T.n_gate[0]), "octree_nodes": SP.tree.n_nodes, "octree_level": OCT_LEVEL}
    assert not sdf_counts["sample_overflow"], sdf_counts

    # end-to-end through the public API with host buffers
    for sl in slots:
        sl["free"].record(torch.cuda.current_stream())
    step_e2e(0, last=True)  # warm the path
    if world > 1:
        pre_render()
    torch.cuda.synchronize()
    ms_e2e = timed(lambda i: step_e2e(i, last=(i == args.steps - 1)), args.steps) / args.steps
    e2e_value = world * 1e3 / ms_e2e
    h2d = 16 * 4 + 9 * 4 + H * W * 4 * 4
    d2h = 4

    # per-stage times of OUR step (CUDA events between the stages of 5 extra steps; outside the timed regions)
    # (world > 1: every rank runs the extra steps -- they contain collectives -- and rank 0 reports; the waits for the two all-reduces
    # then show up inside the stage that issues them: the splat segment's in projection_fwd, the SDF segment's in adam)
    stage_ms = None
    if True:
        acc = {}
        T.overlap = False  # the per-stage table is taken with the stages in line on one stream (event differences are meaningless otherwise)
        for i in range(5):
            R.stage_events = [] if rank == 0 else None
            step_resident(i)
            if world > 1:
                pre_render()
            torch.cuda.synchronize()
            ev = R.stage_events or []
            for (_, a), (name, b) in zip(ev[:-1], ev[1:]):
                acc.setdefault(name, []).append(a.elapsed_time(b))
        R.stage_events = None
        T.overlap = args.overlap > 0 and T.mlp_mode == 1
        stage_ms = {("rng+sample_generation[A0]" if k == "start" else k): float(np.mean(v)) for k, v in acc.items()} if rank == 0 else None

    if rank == 0:
        pk, pk_kind = peaks()
        # SURVEY 8d quotes the algorithmic bytes per REFERENCE intersection (every tile of a splat's radius AABB): I_ref. The fused
        # step drops the pairs whose exact footprint misses the tile before the sort, so the kernels only walk I_kept of them: the
        # roofline fraction is computed on the units the launch processes; the reference-unit figure is a side field.
        nnz, I_kept, I, P = cnt["nnz"], cnt["n_isects"], max(cnt["n_isects_aabb"], cnt["n_isects"]), W * H
        alg_bwd_ref = 148 * I + 64 * P + 8 * nnz   # SURVEY 8d: raster_bwd = 76 I + 64 P + 72 I + 8 nnz
        alg_bwd = 148 * I_kept + 64 * P + 8 * nnz
        alg_fwd = 76 * I_kept + 56 * P + 4 * nnz
        t_bwd = float(np.mean(bwd_ms)) * 1e-3
        t_fwd = float(np.mean(fwd_ms)) * 1e-3
        achieved = alg_bwd / t_bwd / 1e9
        line = {"metric": "train_steps_per_s", "value": value, "unit": "step/s", "n_gpus": world, "steps": args.steps,
                "warmup": max(args.warmup, 3), "ms_per_step": ms_step, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
                "dtype": "f32", "data": "synthetic", "config": cfg, "mrays_per_s": value * P / 1e6, "clocks": clocks,
                "e2e": {"value": e2e_value, "unit": "step/s", "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": d2h,
                        "ms_per_step": ms_e2e},
                # ours only (torch's RNG fills not counted): 30 of GsSdfStep - table cast - weight pack (now inside the Adam call) + normal-consistency
                # + isotropic + Adam + weight pack + 6 sample-generation kernels + octree query + gate compaction (3, replaces the gate count) + row scatter (2) + densify statistics
                # (N > 1 with the sparse exchange: + row pack + one row unpack per rank; NCCL's own kernels are not ours)
                "gpu_launches": args.steps * (render.GsSdfStep.KERNELS_PER_STEP - 2 + 2 + 2 + 7 + 2 + 2 + 1 + ((1 + world) if DP.sparse_steps else 0)),
                "step_contents": "[A] octree ray-march sample generation of 3277 depth rays (~32 k points) + SDF stage on them, [B] render, [C] "
                                 "GS<->SDF coupling gated by visibility and octree validity, [D] L1 + DSSIM + depth L1 + normal-consistency + "
                                 "isotropic -> backward, Adam over all parameter groups, densification statistics (update_state); not in the "
                                 "step: the every-100-iterations grow / split / prune surgery of NeuralGS::train_callback",
                "roofline": {"kernel": "raster2dgs_bwd_kernel", "bound": "hbm", "achieved": achieved, "peak": pk["hbm_gbs"], "unit": "GB/s",
                             "frac": achieved / pk["hbm_gbs"], "peak_source": pk_kind,
                             "algorithmic_bytes": alg_bwd, "kernel_ms": t_bwd * 1e3,
                             "units": {"I_processed": I_kept, "I_reference_aabb": I, "P": P, "nnz": nnz},
                             "frac_on_reference_units": alg_bwd_ref / t_bwd / 1e9 / pk["hbm_gbs"],
                             "note": "frac = SURVEY 8d bytes on the intersections the launch processes (after exact pre-sort culling) / event "
                                     "time / peak HBM bandwidth (peak_source)",
                             "raster_fwd": {"achieved": alg_fwd / t_fwd / 1e9, "frac": alg_fwd / t_fwd / 1e9 / pk["hbm_gbs"],
                                            "kernel_ms": t_fwd * 1e3, "algorithmic_bytes": alg_fwd}},
                "splat_exchange_steps": {"visible_rows": DP.sparse_steps, "dense_allreduce": DP.dense_steps} if world > 1 else None,
                "counts": cnt, "counts_end": cnt_end, "sdf_counts": sdf_counts, "loss_end": last_loss, "loss_finite": bool(np.isfinite(last_loss)),
                "stage_ms": stage_ms,
                # every device buffer of the library is a torch tensor, so the allocator's peak is the workload's footprint
                "device_memory_peak_gib": torch.cuda.max_memory_allocated(dev) / 2 ** 30}
        if world == 1 and not args.no_stock_cuda:
            try:
                line["stock_cuda"] = run_stock_cuda(torch, S, sc_act, cams, gts, W, H, deg, dev, stage_ms, steps=args.steps)
            except Exception as e:  # test infrastructure missing on this box: say so, never fail the bench
                line["stock_cuda"] = {"unavailable": f"{type(e).__name__}: {e}"[:300]}
        if world == 1 and not args.no_cpu_baseline:
            cb = run_cpu_c1()
            try:  # the same c1 step on this GPU: a measured like-for-like pair
                del T
                torch.cuda.empty_cache()
                W1, H1, N1, deg1, _ = WORKLOADS["c1"]
                T1, act1, _ = build_trainer("c1", args.eikonal)
                SP1 = Sampling(T1, act1["means"], 50)
                cams1 = [S.camera(i, W1, H1) for i in range(n_cams)]
                gts1 = gt_images(T1, act1, cams1, W1, H1)
                dc1 = [(t(V_[None]), t(K_[None])) for V_, K_ in cams1]
                rb1 = torch.empty(N1, 2, device=dev)

                def c1_step(i):
                    rb1.normal_()
                    rx, rg, rc = SP1.draw(i)
                    T1.train_step(dc1[i % n_cams][0], dc1[i % n_cams][1], gts1[i % n_cams], rx, rg, rb1, ray_n_live=rc)
                    T1.adam_all()
                for i in range(5):
                    c1_step(i)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for i in range(args.steps):
                    c1_step(i)
                e1.record()
                torch.cuda.synchronize()
                gpu_c1 = args.steps * 1e3 / e0.elapsed_time(e1)
                cb["gpu_same_config"] = {"value": gpu_c1, "unit": "step/s", "ms_per_step": 1e3 / gpu_c1, "steps": args.steps,
                                         "counts": T1.R.read_counts(), "ratio_gpu_over_cpu": gpu_c1 / cb["value"]}
            except Exception as e:
                cb["gpu_same_config"] = {"unavailable": f"{type(e).__name__}: {e}"[:300]}
            line["cpu_baseline"] = cb
        print(json.dumps(line))
    if world > 1:
        dist.destroy_process_group()
    return 0


def dump_outputs(out_dir, arrays, budget=60 << 20):
    """Writes each array as out_dir/<name>.npy in float32. An array larger than its equal share of `budget` bytes is replaced by the
    elements at a fixed, seeded set of flat indices (sorted; the same set for the same array size), so that two builds run with the same
    arguments can be compared output for output."""
    os.makedirs(out_dir, exist_ok=True)
    share = budget // 4 // len(arrays)
    for name, a in arrays.items():
        a = a.detach().float().cpu().numpy()
        if a.size > share:
            a = a.reshape(-1)[np.sort(np.random.default_rng(0).choice(a.size, share, replace=False))]
        np.save(os.path.join(out_dir, name + ".npy"), np.ascontiguousarray(a, dtype=np.float32))


def run_stock_cuda(torch, S, sc_act, cams, gts, W, H, deg, dev, ours_stage_ms, steps=5):
    """The reference fork's own kernels (projection -> SH -> tile_encode incl. its CUB sort -> raster fwd -> raster bwd -> SH bwd ->
    projection bwd, host glue of oracle/ref_driver.cpp incl. the reference's .item() syncs) on the SAME activated tensors, CUDA events per
    stage, median of `steps` runs after two warm-ups. Test infrastructure: imported here and nowhere in the product path."""
    import importlib
    ref_dir = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.exists(os.path.join(ref_dir, "gsplat_ref.so")):
        return {"unavailable": "oracle/_ref/gsplat_ref.so not built (python oracle/build_ref.py where /root/reference exists)"}
    if ref_dir not in sys.path:
        sys.path.insert(0, ref_dir)
    ref = importlib.import_module("gsplat_ref")
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    means, quats, scales, sh, opac = sc_act["means"], sc_act["quats"], sc_act["scales"], sc_act["sh"], sc_act["opacities"]
    N = means.shape[0]
    tw, th = (W + 15) // 16, (H + 15) // 16
    names = ["projection_fwd", "sh_fwd", "tile_encode", "raster_fwd", "raster_bwd", "sh_bwd", "projection_bwd"]
    acc = {k: [] for k in names}
    info = {}
    warm = 2  # the first calls grow torch's caching allocator (cudaMalloc inside the stages)
    for it in range(steps + warm):
        V, Kc = cams[it % len(cams)]
        Vt, Kt = t(V[None]), t(Kc[None])
        gt = gts[it % len(gts)]
        rn = torch.randn(N, 2, device=dev)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(names) + 1)]
        ev[0].record()
        (indptr, cam, gid, radii, m2d, dep, rt, nrm, randns, samples) = ref.projection_2dgs_packed_fwd(
            means, quats, scales, Vt, Kt, W, H, S.NEAR, S.FAR, 0.0, rn)
        ev[1].record()
        c2w = torch.inverse(Vt)  # get_view_colors (GSC/rendering.cpp:27-44)
        dirs = (means[gid] - c2w[cam, :3, 3]).contiguous()
        shs = sh[gid].contiguous()
        sh_raw = ref.sh_fwd(deg, dirs, shs)
        colors = torch.clamp_min(sh_raw + 0.5, 0.0).contiguous()
        pt_op = opac[gid].contiguous()
        ev[2].record()
        tpg, isect_ids, flatten_ids, offsets = ref.tile_encode(m2d, radii, dep, cam, gid, 1, 16, tw, th)
        ev[3].record()
        fw = ref.raster_fwd(m2d, rt, colors, pt_op, nrm, W, H, 16, offsets, flatten_ids)
        (r_col, r_dep, r_alp, r_Ts, r_nrm, r_dis, r_med, last_ids, median_ids, vis) = fw
        ev[4].record()
        npx = float(W * H)
        v_col = torch.sign(r_col - gt[..., :3]) / (3 * npx)
        v_dep = torch.sign(r_dep / r_alp.clamp_min(1e-8) - gt[..., 3:]) * 0.1 / npx
        z1, z3 = torch.zeros_like(r_alp), torch.zeros_like(r_nrm)
        bw = ref.raster_bwd(m2d, rt, colors, pt_op, nrm, W, H, 16, offsets, flatten_ids, r_col, r_dep, r_alp, r_Ts, last_ids, median_ids,
                            v_col.contiguous(), v_dep.contiguous(), z1, z3, z1, z1)
        torch.cuda.synchronize()  # GSC/rasterize_to_pixels.cpp:252: the reference synchronises after its raster backward
        ev[5].record()
        v_m2d, v_rt, v_colr, v_op, v_nrm, v_den = bw
        v_coeffs, v_dirs = ref.sh_bwd(deg, dirs, shs, (v_colr * (sh_raw + 0.5 > 0)).contiguous())
        v_sh = torch.zeros_like(sh).index_add_(0, gid, v_coeffs)  # the ATen index backward of the gathers
        ev[6].record()
        pb = ref.projection_2dgs_packed_bwd(means, quats, scales, Vt, Kt, W, H, cam, gid, rt, randns, v_m2d, torch.zeros_like(dep), v_rt,
                                            v_nrm, torch.zeros_like(samples))
        ev[7].record()
        torch.cuda.synchronize()
        if it >= warm:
            for k, a, b in zip(names, ev[:-1], ev[1:]):
                acc[k].append(a.elapsed_time(b))
        info = {"nnz": int(gid.shape[0]), "n_isects": int(flatten_ids.shape[0])}
    st = {k: float(np.median(v)) for k, v in acc.items()}  # median: a stray cudaMalloc in one run must not colour the stage table
    total = float(sum(st.values()))
    out = {"kind": "reference fork CUDA kernels (gsplat 2DGS path of GS-SDF) compiled for sm_90a with the reference's flags (-O3 "
                   "--use_fast_math), same GPU, same tensors", "stage_ms": st, "splat_chain_ms": total, "steps": steps, "counts": info,
           "covers": "splat chain only (a2-a7): no losses, no SDF stages, no optimiser"}
    if ours_stage_ms:
        mine = {k: ours_stage_ms.get(k) for k in names}
        if all(v is not None for v in mine.values()):
            out["ours_stage_ms"] = mine
            out["ours_splat_chain_ms"] = float(sum(mine.values()))
            out["speedup_splat_chain"] = total / out["ours_splat_chain_ms"]
            out["speedup_per_stage"] = {k: st[k] / mine[k] for k in names if mine[k] > 0}
    return out


if __name__ == "__main__":
    sys.exit(main())
