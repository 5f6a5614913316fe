"""The SDF pre-training stage of GS-SDF, NeuralSLAM::nsdf_train (include/neural_mapping/neural_mapping.cpp:294-354), on the GPU without host
synchronisation (row f-13, DESIGN 7n).

Per iteration the reference draws k_batch_num rays of the training depth pack (sdf_train_batch_iter, :143-156), samples them with the sample
std k_sample_std, trains the SDF on the samples (BCE + analytic eikonal + align, whose numerical gradient uses the offset k_sample_std), steps
Adam, and then adapts three quantities (:324-330, sdf_train_callback :533-593): the ray count follows an EMA of the samples per ray so that a
batch holds about k_batch_pt_num points, k_sample_std becomes max(mean(1 / isigma), k_bce_sigma), and the learning rate runs linearly from lr
to lr_end. The reference reads the count and the mean back with .item() every iteration; `SdfTrainer` keeps them on the device
(gssdf_sdf_adapt) where the batch draw (gssdf_sdf_ray_batch), the sampler (gssdf_sdf_sample_rays_dev) and the SDF kernels
(gssdf_sdf_fwd_dev / gssdf_sdf_train_dev) read them. Only the learning rate is a host scalar (a function of the iteration alone).

Deliberate departures: the rays are drawn from a device generator (the reference uses a CPU torch::rand: same distribution, another stream);
the sample std is a deterministic fp64-accumulated mean (the reference's fp32 ATen mean may differ in the last bit).
"""

import numpy as np
import torch

from . import cabi
from . import octree as OT
from . import sdf as SD

PACK_KEYS = ("origin", "direction", "depth", "xyz")
_f32 = np.float32


# ---- host restatements of the reference's scalar rules (checked against the compiled C++ in tests/test_nsdf_host.py) ----------------
def initial_state(batch_pt_num):
    """params.cpp:198-204 and nsdf_train's first lines (:298-299): (sample_std = bce_sigma is set by the caller), n_rays = (int)batch_pt_num,
    pts_per_ray = batch_pt_num / (float)n_rays in fp32. Returns (pts_per_ray, n_rays)."""
    b = _f32(batch_pt_num)
    n = int(b)
    return _f32(b / _f32(n)), n


def adapt_rays(pts_per_ray, n_rays, pt_n, batch_pt_num):
    """nsdf_train :324-330 in the reference's types: sample_pts_per_ray = (float)pt_n / (float)n_rays (fp32), the EMA in double rounded to
    float, n_rays = (int)min(batch_pt_num / pts_per_ray, batch_pt_num) with the division in fp32 and the min taken in float (equal to the
    reference's min((int)q, (int)batch_pt_num) wherever (int)q is defined). Returns (pts_per_ray, n_rays)."""
    b = _f32(batch_pt_num)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        spr = _f32(_f32(pt_n) / _f32(n_rays))
        ppr = _f32(float(_f32(pts_per_ray)) * 0.9 + float(spr) * 0.1)
        q = _f32(b / ppr)
    m = q if q < b else b
    return ppr, int(m)


def lr_at(it, total_it, lr, lr_end):
    """sdf_train_callback :550-557: lr * (1 - r) + lr_end * r with r = (float)it / total_it, all fp32 (the rate of the NEXT iteration)."""
    r = _f32(it) / _f32(total_it)
    return float(_f32(_f32(lr) * (_f32(1) - r)) + _f32(_f32(lr_end) * r))


def ray_index(rand, N):
    """The batch draw's index rule (:145-152): (rand * N).to(kLong).clamp(0, N - 1) with N rounded to fp32 (float32 numpy in, int64 out)."""
    p = np.asarray(rand, _f32) * _f32(N)
    return np.clip(p.astype(np.int64), 0, N - 1)


def new_adapt_state(device, bce_sigma, batch_pt_num):
    """The device state of gssdf_sdf_adapt, {float sample_std, float pts_per_ray, int32 n_rays, pad}, as an int32 CUDA tensor [4]."""
    ppr, n = initial_state(batch_pt_num)
    raw = np.zeros(4, np.int32)
    raw[:2] = np.array([bce_sigma, ppr], _f32).view(np.int32)
    raw[2] = n
    return torch.from_numpy(raw).to(device)


def read_state(state):
    """(sample_std, pts_per_ray, n_rays) of a device state (one read-back)."""
    raw = state.cpu().numpy()
    f = raw[:2].view(_f32)
    return float(f[0]), float(f[1]), int(raw[2])


class SdfTrainer:
    """nsdf_train on a device-resident depth pack: `step(i)` enqueues iteration i with no host synchronisation (except the kept-row count
    of an outlier-removal iteration); `histories()` reads the per-iteration loss, sample std, ray count and sample count once at the end.

    net: an sdf.SdfNet with the tensor-core decoder (hidden 64, 3 hidden layers; its parameters are copied in). tree: the occupancy
    OctreeAS (octree.build_occ_map). pack: dict of float32 CUDA tensors origin [N,3], direction [N,3] (unit), depth [N] or [N,1], xyz [N,3]
    (the layout of base_parser.cpp:925-960). xyz_min / xyz_max: the SubMap's in-range box in world units (pos_W_M + xyz_min_M / xyz_max_M).
    Supported configuration: the one every shipped config uses (config/base.yaml): analytic eikonal, curvature weight 0."""

    def __init__(self, net, tree, pack, iters, *, leaf_size, bce_sigma, xyz_min, xyz_max, lr=5e-3, lr_end=1e-4, batch_pt_num=32768,
                 sdf_weight=1.0, eikonal_weight=0.1, align_weight=0.1, curvate_weight=0.0, numerical_grad=False, n_free=3, n_surface=3,
                 outlier_remove=False, outlier_dist=0.05, outlier_interval=2000, vis_batch_pt_num=1_638_400, nugget_per_ray=16, seed=0):
        if numerical_grad:
            raise ValueError("SdfTrainer: numerical_grad 1 is not supported (the trainer runs the analytic eikonal of config/base.yaml)")
        if curvate_weight != 0.0:
            raise ValueError("SdfTrainer: curvate_weight must be 0 (config/base.yaml); the curvature term is not implemented")
        if net.mlp_mode != 1 or net.cfg["hidden_dim"] != 64 or net.cfg["n_hidden"] != 3:
            raise ValueError("SdfTrainer: needs the tensor-core decoder (mlp_mode 1, hidden_dim 64, geo_num_layer 3)")
        if not (align_weight >= 0.0 and iters >= 1 and batch_pt_num >= 1):
            raise ValueError("SdfTrainer: align_weight >= 0, iters >= 1 and batch_pt_num >= 1 are required")
        dev = net.params_.device
        for k in PACK_KEYS:
            t = pack[k]
            if not (t.is_cuda and t.dtype == torch.float32 and t.device == dev):
                raise ValueError(f"SdfTrainer: pack[{k!r}] must be a float32 tensor on {dev}")
        self.dev, self.iters, self.net_mod = dev, int(iters), net
        self.cfg = dict(net.cfg)
        self.lr0, self.lr_end, self.lr = float(lr), float(lr_end), float(lr)
        self.bce_sigma = float(_f32(bce_sigma))
        self.bce_isigma = float(_f32(1.0) / _f32(bce_sigma))  # k_bce_isigma = 1.0f / k_bce_sigma
        self.truncated_dis = float(_f32(3) * _f32(leaf_size))  # k_truncated_dis = 3 * k_leaf_size
        self.batch_pt_num = float(_f32(batch_pt_num))
        self.sdf_w, self.eik_w, self.align_w = float(sdf_weight), float(eikonal_weight), float(align_weight)
        self.outlier_remove, self.outlier_dist, self.outlier_interval = bool(outlier_remove), float(outlier_dist), int(outlier_interval)
        self.vis_batch_pt_num = int(vis_batch_pt_num)
        # parameters: ONE flat [table | decoder] buffer with Adam's moments and gradient of the same layout
        self.n_table, self.n_mlp = net.params_.numel(), net.decoder_.numel()
        f32 = dict(dtype=torch.float32, device=dev)
        self.params = torch.cat([net.params_.detach().reshape(-1), net.decoder_.detach().reshape(-1)]).contiguous()
        self.exp_avg, self.exp_avg_sq, self.grad = torch.zeros_like(self.params), torch.zeros_like(self.params), torch.zeros_like(self.params)
        self.table, self.mlp = self.params[:self.n_table], self.params[self.n_table:]
        self.table_grad, self.mlp_grad = self.grad[:self.n_table], self.grad[self.n_table:]
        self.table_half = torch.empty(self.n_table, dtype=torch.float16, device=dev)
        probe = cabi.sdf_net(self.table_half, self.mlp, **self.cfg)
        self.mlp_packed = torch.empty(cabi.sdf_mlp_packed_bytes(probe), dtype=torch.uint8, device=dev)
        self.net = cabi.sdf_net(self.table_half, self.mlp, origin=net.origin, inv_size=net.inv_size, mlp_mode=1, mlp_packed=self.mlp_packed,
                                **self.cfg)
        cabi.sdf_table_to_half(self.table, self.table_half)
        cabi.sdf_mlp_pack(self.net, self.mlp_packed)
        # the pack, double-buffered for the outlier compaction
        self.N = int(pack["xyz"].shape[0])
        if self.N < 1:
            raise ValueError("SdfTrainer: the pack is empty")
        self._pack = {k: pack[k].reshape(self.N, -1).contiguous().clone() for k in PACK_KEYS}
        self._pack_alt = None
        # the batch: ray capacity = the largest ray count gssdf_sdf_adapt can set, (int)batch_pt_num
        self.ray_cap = int(self.batch_pt_num)
        self.rand = torch.empty(self.ray_cap, **f32)
        self.rays = {k: torch.empty(self.ray_cap, 1 if k == "depth" else 3, **f32) for k in PACK_KEYS}
        self.rs = OT.RaySampler(tree, self.ray_cap, dev, 1, n_free, n_surface, sample_std=self.bce_sigma, truncated_dis=self.truncated_dis,
                                xyz_min=tuple(xyz_min), xyz_max=tuple(xyz_max), nugget_cap=nugget_per_ray * self.ray_cap)
        cap = self.rs.cap
        nv = 7 if self.align_w > 0 else 1
        self.s_var, self.y_var = torch.empty(nv * cap, **f32), torch.empty(nv * cap, **f32)
        # device state {sample_std, pts_per_ray, n_rays}; the sampler / SDF kernels read sample_std, the draw reads n_rays
        self.adapt = new_adapt_state(dev, self.bce_sigma, self.batch_pt_num)
        self.std_dev = self.adapt.view(torch.float32)[0:1]
        self.n_rays_dev = self.adapt[2:3]
        # device histories, read once by histories(): the loss of iteration i, the state after it, its sample count
        self.h_loss = torch.zeros(self.iters, **f32)
        self.h_state = torch.zeros(self.iters, 4, dtype=torch.int32, device=dev)
        self.h_samples = torch.zeros(self.iters, dtype=torch.int32, device=dev)
        self.overflow = torch.zeros(1, dtype=torch.int32, device=dev)  # the sampler's overflow flag, latched over all iterations
        self.gen = torch.Generator(dev).manual_seed(seed)
        self.ws = cabi.Workspace(dev)
        self.n_kept = torch.zeros(1, dtype=torch.int64, device=dev)
        self.t = 0  # Adam steps taken

    @property
    def pack(self):
        return {k: v[:self.N] for k, v in self._pack.items()}

    def sdf_groups(self, lr):
        """GsSdfTrainer.sdf_groups' layout: the table (with its fp16 shadow refreshed) and the decoder, at one learning rate."""
        return [(0, self.n_table, lr, True), (self.n_table, self.n_mlp, lr, False)]

    def draw(self):
        """The random inputs of one iteration: the ray draw (the reference's torch::rand, :145) and the sampler's rand / randn."""
        self.rand.uniform_(generator=self.gen)
        self.rs.rand_voxel.uniform_(generator=self.gen)
        self.rs.rand_free.uniform_(generator=self.gen)
        self.rs.randn_surface.normal_(generator=self.gen)

    def step(self, i):
        self.draw()
        self.train(i)

    def train(self, i):
        """Iteration i on the drawn inputs, in the reference's order: batch draw, sampling, 7-variant forward (y1 of the base rows for the
        sample std; the six offsets for the align loss), fused BCE + eikonal + align train kernel, Adam at the current rate, state update,
        next rate, and at i > 0 && i % interval == 0 the outlier removal (when enabled)."""
        rs = self.rs
        cabi.sdf_ray_batch(self.pack, self.rand, self.n_rays_dev, self.rays)
        rs.sample(self.rays["origin"], self.rays["direction"], self.rays["depth"], self.rays["xyz"], n_live=self.n_rays_dev,
                  sample_std=self.std_dev)
        torch.bitwise_or(self.overflow, rs.counts[2:3], out=self.overflow)
        n_live = rs.counts  # counts[0]: samples of this iteration
        align = self.align_w > 0
        cabi.sdf_fwd_dev(self.net, rs.xyz, self.s_var, self.std_dev, y1=self.y_var, n_variants=7 if align else 1, n_live=n_live)
        cabi.sdf_train_dev(self.net, rs.xyz, 1, self.std_dev, rs.ray_sdf, None, self.bce_isigma, self.sdf_w, self.eik_w, 0.0,
                           self.h_loss[i:i + 1], self.table_grad, self.mlp_grad, None, n_live=n_live, eikonal_mode=1,
                           align_weight=self.align_w, sdf_variants=self.s_var if align else None)
        self.t += 1
        cabi.adam_step(self.params, self.grad, self.exp_avg, self.exp_avg_sq, self.sdf_groups(self.lr), self.t, eps=1e-15, zero_grads=True,
                       table_half=self.table_half, net=self.net, mlp_packed=self.mlp_packed)
        cabi.sdf_adapt(self.adapt, self.y_var[:rs.cap], n_live, self.bce_sigma, self.bce_isigma, self.batch_pt_num, update_rays=True)
        self.h_state[i].copy_(self.adapt)
        self.h_samples[i:i + 1].copy_(rs.counts[0:1])
        self.lr = lr_at(i, self.iters, self.lr0, self.lr_end)
        if self.outlier_remove and i > 0 and i % self.outlier_interval == 0:
            self.remove_outliers(i)

    def remove_outliers(self, i, total_iter=None, net=None, outlier_dist=None):
        """sdf_train_callback's outlier branch on the device pack (sdf.remove_outliers' rule: threshold and rows from sdf.outlier_threshold /
        sdf.outlier_rows, compaction by gssdf_sdf_outlier_filter into the second pack buffer). Reads the kept count once. total_iter / net /
        outlier_dist default to this stage's; the joint stage (gstrain) passes its iteration count, its SDF and its setting."""
        thr = SD.outlier_threshold(i, self.iters if total_iter is None else total_iter, self.truncated_dis,
                                   self.outlier_dist if outlier_dist is None else outlier_dist)
        n = SD.outlier_rows(self.N, self.vis_batch_pt_num)
        if self._pack_alt is None:
            self._pack_alt = {k: torch.empty_like(v) for k, v in self._pack.items()}
        cols = [(self._pack[k], self._pack_alt[k]) for k in PACK_KEYS]
        cabi.sdf_outlier_filter(self.net if net is None else net, self._pack["xyz"], thr, cols, self.n_kept, self.ws, n=n)
        kept = int(self.n_kept.item())
        if kept < 1:
            raise RuntimeError(f"SdfTrainer: the outlier removal of iteration {i} (threshold {thr:g}) kept no row of the pack")
        self._pack, self._pack_alt = self._pack_alt, self._pack
        self.N = kept

    def run(self, start=0, stop=None):
        for i in range(start, self.iters if stop is None else stop):
            self.step(i)

    def histories(self):
        """Per-iteration device histories, read once: loss, sample_std / pts_per_ray / n_rays after the iteration's update, sample count.
        Raises if the sampler's capacity overflowed in any iteration."""
        if int(self.overflow.item()):
            raise RuntimeError("SdfTrainer: the ray sampler's sample or nugget capacity overflowed (raise nugget_per_ray)")
        st = self.h_state.cpu().numpy()
        f = np.ascontiguousarray(st[:, :2]).view(_f32)
        return dict(loss=self.h_loss.cpu().numpy(), sample_std=f[:, 0].copy(), pts_per_ray=f[:, 1].copy(), n_rays=st[:, 2].copy(),
                    n_samples=self.h_samples.cpu().numpy())

    def state(self):
        """(table, mlp, sample_std) for GsSdfTrainer.load(..., table, mlp) / GsSdfTrainer(delta=sample_std): the trained parameters (views
        of the flat buffer) and the sample std after the last iteration (read back once)."""
        return self.table, self.mlp, read_state(self.adapt)[0]

    def write_back(self):
        """Copy the trained parameters into the SdfNet the trainer was built from (for mesh.meshing, sdf.remove_outliers, ...)."""
        with torch.no_grad():
            self.net_mod.params_.copy_(self.table)
            self.net_mod.decoder_.copy_(self.mlp)
        return self.net_mod

    def __repr__(self):
        return f"SdfTrainer(N={self.N}, iters={self.iters}, ray_cap={self.ray_cap}, sample_cap={self.rs.cap})"
