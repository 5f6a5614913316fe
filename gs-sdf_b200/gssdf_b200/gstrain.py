"""The joint stage of GS-SDF, NeuralSLAM::gs_train (include/neural_mapping/neural_mapping.cpp:356-531), on the GPU with its state kept on
the device (DESIGN 7o).

`GsTrainer` continues from a finished `nsdf.SdfTrainer`: it takes over its net, occupancy tree, sampler, depth pack (with the outlier
double buffer), the adaptive state {sample_std, pts_per_ray, n_rays} and the SDF parameters with their Adam moments and step count, and
runs the reference's loop in the reference's order:

  colour initialisation (color_init): train_num iterations at SH degree 0 with the photometric loss only, the structure frozen and the SH
      groups stepped at 10x rate on their own Adam clock; afterwards every rate is lr * 10 * (double)0.1f, as the reference leaves it;
  the rate-only effect of train_callback(0, ..., empty_map): offsets at 1.6e-4 * spatial_scale, SDF at min(that, lr_end);
  gs_iter_step joint iterations: camera draw, SDF ray batch, sampling with the device sample std, the joint step with the device sample
      std at both SDF sites, one Adam launch over every group at its own clock, sdf_train_callback (sample std only, ray count frozen;
      outlier removal when due), and for i < gs_iter_step / 2 Densifier.train_callback (the reference's early return), whose SH degree
      the next render uses.

Deliberate departures: the camera permutation comes from a seeded torch CPU generator (same distribution, another stream); the sample std
is an fp64-accumulated mean (nsdf); colour initialisation skips the projection backward, whose gradients the reference computes and
discards; the per-iteration logged values are device histories read once; Densifier's learning rate is computed in double."""
import math

import numpy as np
import torch

from . import cabi
from . import densify as DN
from . import render as RD
from . import sdf as SD

_f32 = np.float32


# ---- the loop's host rules (checked against the reference's expressions compiled with g++ in tests/test_gs_train_host.py) -------------
def color_init_lr(lr):
    """The rate a group keeps after colour initialisation: set_lr(10 * lr), then set_lr(0.1f * lr) in double (neural_mapping.cpp:373,384)."""
    return (10 * lr) * float(_f32(0.1))


def xyz_lr(it, total_iter, spatial_scale):
    """The offsets' rate Densifier.train_callback sets at iteration `it` (neural_gaussian.cpp:604-623, in double as Densifier computes it)."""
    ratio = it / float(total_iter)
    lr0, lr1 = 1.6e-4 * spatial_scale, 1.6e-6 * spatial_scale
    return math.exp(math.log(lr0) * (1 - ratio) + math.log(lr1) * ratio)


def callback_due(i, total_iter):
    """NeuralGS::train_callback acts (densification, SH degree, rate decay) only below refine_stop_iter = total / 2 (:574-579)."""
    return i < total_iter // 2


def normal_on(i, refine_gs_struct_start_iter):
    """The normal-consistency term of joint iteration i (neural_mapping.cpp:244-245)."""
    return i > refine_gs_struct_start_iter


def perm_due(i, train_num):
    """A fresh randperm(train_num) before iteration i (neural_mapping.cpp:205-212)."""
    return i % train_num == 0


def adam_clocks(i, sdf_steps, train_num, color_init):
    """The Adam step counts of joint iteration i: (SDF groups, SH groups, other splat groups)."""
    return sdf_steps + i + 1, train_num * int(bool(color_init)) + i + 1, i + 1


def outlier_due(i, interval):
    return i > 0 and i % interval == 0


class FramesU8:
    """8-bit RGB training frames of any sizes packed in one uint8 buffer (DESIGN 7q): frame i is sizes[i] = (W_i, H_i), W_i H_i 3 bytes of
    interleaved RGB at byte offsets[i]. `data` lives on the device or in pinned host memory; GsTrainer expands one frame per iteration
    on the device into the loss's float ground truth as the reference's convertTo(CV_32FC3, 1.0f / 255.0f) does (gssdf_frames_u8_expand),
    after copying only that frame's bytes when the store is pinned. A quarter of the bytes of float frames."""

    def __init__(self, data, sizes):
        self.sizes = [(int(w), int(h)) for w, h in sizes]
        if not self.sizes or min(min(wh) for wh in self.sizes) < 1:
            raise ValueError("FramesU8: at least one frame, every width and height >= 1")
        if not (isinstance(data, torch.Tensor) and data.dtype == torch.uint8 and data.dim() == 1 and data.is_contiguous()):
            raise ValueError("FramesU8: data must be a contiguous uint8 tensor [n_bytes]")
        self.offsets = np.concatenate([[0], np.cumsum([3 * w * h for w, h in self.sizes])]).astype(np.int64).tolist()
        if data.numel() != self.offsets[-1]:
            raise ValueError(f"FramesU8: {len(self.sizes)} frames need {self.offsets[-1]} bytes, data has {data.numel()}")
        self.data = data

    @classmethod
    def pack(cls, frames, device=None, pin=False):
        """frames: uint8 [H_i,W_i,3] RGB arrays or tensors. The store goes to `device`, or to pinned host memory with pin=True."""
        ts = [torch.as_tensor(np.ascontiguousarray(f) if isinstance(f, np.ndarray) else f) for f in frames]
        for t in ts:
            if t.dtype != torch.uint8 or t.dim() != 3 or t.shape[-1] != 3:
                raise ValueError("FramesU8.pack: every frame must be uint8 [H,W,3]")
        data = torch.cat([t.reshape(-1).cpu() for t in ts]) if ts else torch.zeros(0, dtype=torch.uint8)
        data = data.pin_memory() if pin else data.to(device) if device is not None else data
        return cls(data, [(int(t.shape[1]), int(t.shape[0])) for t in ts])

    @property
    def is_cuda(self):
        return self.data.is_cuda

    def frame(self, i):
        """Frame i as uint8 [H,W,3] (a view of the store)."""
        w, h = self.sizes[i]
        return self.data[self.offsets[i]:self.offsets[i + 1]].view(h, w, 3)


def parse_frames(images):
    """GsTrainer's `images`: ("stack", [(W,H)] * T) for a float32 [T,H,W,3] tensor (the path of one camera), ("list", sizes) for a list
    of float32 [H_i,W_i,3] tensors, ("u8", sizes) for a FramesU8 store. Shapes only: where the frames live is checked later."""
    if isinstance(images, FramesU8):
        return "u8", list(images.sizes)
    if isinstance(images, (list, tuple)):
        if not images:
            raise ValueError("GsTrainer: the list of frames is empty")
        for t in images:
            if not (isinstance(t, torch.Tensor) and t.dtype == torch.float32 and t.dim() == 3 and t.shape[-1] == 3 and t.shape[0] >= 1
                    and t.shape[1] >= 1):
                raise ValueError("GsTrainer: every frame of a list must be a float32 tensor [H,W,3]")
        return "list", [(int(t.shape[1]), int(t.shape[0])) for t in images]
    if not (isinstance(images, torch.Tensor) and images.dtype == torch.float32 and images.dim() == 4 and images.shape[-1] == 3):
        raise ValueError("GsTrainer: images must be a float32 tensor [T,H,W,3], a list of float32 [H,W,3] tensors or a FramesU8 store")
    return "stack", [(int(images.shape[2]), int(images.shape[1]))] * int(images.shape[0])


class GsTrainer:
    """gs_train on the device. `run()` runs colour initialisation (when enabled) and the gs_iter_step joint iterations; `histories()` reads
    the per-iteration device records once; `state()` returns what mesh.meshing, io.export_gs_to_ply and metrics.eval_render take.

    sdf: an nsdf.SdfTrainer that has finished its stage (its state moves here; do not step it afterwards).
    splats: the dict gs_init.neural_gs_init / neural_gs_init_points return (anchors, offsets, quaternion, scaling, opacity, features_dc,
        features_rest), CUDA float32; capacity: the row capacity densification may grow to (rounded up to a multiple of 4).
    poses: [T,4,4] camera-to-world (OpenCV axes); K: [3,3] pinhole shared by every frame, or [T,3,3] a camera per frame (DESIGN 7q);
        images: float32 [T,H,W,3] in [0,1], a list of T float32 [H_i,W_i,3] (frames of several sizes), or a FramesU8 store of 8-bit
        frames expanded on the device; on the device or in pinned host memory (then one frame is copied per iteration, asynchronously).
        Each frame is rendered at its own size with its own K (projection, normal term, background); the densifier's radii normaliser
        is the first trained frame's max(W, H), as in the reference. The reference resizes every ground-truth frame to its first
        camera's size, so it trains cameras of one size only; several sizes are an extension here, and nothing is resized.
    spatial_scale: 0.5 * inner_map_size. The remaining keywords are config/base.yaml's keys with its defaults; `densify` holds Densifier's
    keywords (prune_opa .. sh_degree_interval; sh_degree and sh_degree_interval are passed through from here).
    bck_color: the scene's k_bck_color, the background every render composites (colour initialisation, joint iterations, render()):
        0 black, 1 white (FAST-LIVO2, Oxford Spires, HKU), 2 a uniform random image drawn before every render from a device generator of
        its own (`bg_gen`, seeded from `seed`; the splat samples' draws stay those of modes 0 and 1).
    mask: the dataset's image mask, bool or uint8 [H,W], [H,W,1] or [H,W,3] on the device (nonzero = keep), applied to every frame's L1
        and DSSIM terms as loss::rgb_loss / dssim_loss do; the reference has one mask, so every frame must then have its size.
    depth_type: the config's `depth_type` (k_depth_type), the depth the normal-consistency term differentiates from iteration
        refine_gs_struct_start_iter on: 0 the expected depth, any other int the rasteriser's median depth (bounded scenes; the COLMAP
        configurations set 1 or 3)."""

    def __init__(self, sdf, splats, poses, K, images, *, capacity, spatial_scale, gs_iter_step=30000, color_init=True,
                 detach_sdf_grad=False, refine_gs_struct_start_iter=3000, rgb_weight=0.8, dssim_weight=0.2, render_normal_weight=0.01,
                 isotropic_weight=0.05, gs_sdf_weight=1e-3, visible_thr=0.1, outlier_remove=False, outlier_dist=0.05,
                 outlier_removal_interval=2000, sh_degree=3, sh_degree_interval=1000, densify=None, isect_cap=None, seed=0, bck_color=0,
                 mask=None, depth_type=0):
        dev = sdf.dev
        if not (gs_iter_step >= 1 and outlier_removal_interval >= 1 and sh_degree_interval >= 1):
            raise ValueError("GsTrainer: gs_iter_step, outlier_removal_interval and sh_degree_interval must be >= 1")
        is_4d = isinstance(images, torch.Tensor) and images.dim() == 4
        kind, sizes = parse_frames(images) if not is_4d or images.shape[-1] == 3 else (None, [])
        K_shape = tuple(torch.as_tensor(K).shape)
        if kind is not None and K_shape not in ((3, 3), (len(sizes), 3, 3)):
            raise ValueError(f"GsTrainer: K must be [3,3] or [T,3,3] with T = {len(sizes)} frames, got {K_shape}")
        if mask is not None and len(set(sizes)) > 1:
            raise ValueError("GsTrainer: an image mask needs every frame at its size, and the frames have several sizes")
        hw = tuple(images.shape[1:3]) if is_4d else (sizes[0][1], sizes[0][0]) if sizes else (None, None)
        RD.check_photometric("GsTrainer", bck_color, mask, hw[0], hw[1], dev)
        RD.check_depth_type("GsTrainer", depth_type)
        for k in ("xyz", "origin", "direction", "depth"):
            if not sdf.pack[k].is_cuda:
                raise ValueError(f"GsTrainer: the SdfTrainer's pack[{k!r}] must be on the device")
        if kind is None:
            parse_frames(images)  # raises: a 4-D tensor that is not [T,H,W,3]
        store = images.data if kind == "u8" else images
        for t in (store if kind == "list" else [store]):
            if not (t.is_cuda or t.is_pinned()):
                raise ValueError("GsTrainer: images must be on the device or in pinned host memory")
        n_frames = len(sizes)
        W, H = sizes[0]
        poses = torch.as_tensor(poses)
        if n_frames < 1 or tuple(poses.shape) != (n_frames, 4, 4):
            raise ValueError(f"GsTrainer: poses must be [{n_frames},4,4] for {n_frames} images, got {tuple(poses.shape)}")
        n0 = int(splats["anchors"].shape[0])
        if not 1 <= n0 <= capacity:
            raise ValueError(f"GsTrainer: {n0} initial splats do not fit a capacity of {capacity}")
        self.sdf, self.dev, self.iters, self.train_num = sdf, dev, int(gs_iter_step), n_frames
        self.color_init, self.detach = bool(color_init), bool(detach_sdf_grad)
        self.refine_struct_start, self.normal_w = int(refine_gs_struct_start_iter), float(render_normal_weight)
        self.depth_type = depth_type
        self.outlier_remove, self.outlier_dist, self.outlier_interval = bool(outlier_remove), float(outlier_dist), int(outlier_removal_interval)
        self.spatial_scale = float(spatial_scale)
        self.viewmats = torch.linalg.inv(poses.to(torch.float64)).to(torch.float32).to(dev).contiguous()
        Kt = torch.as_tensor(K, dtype=torch.float32)
        self.Ks = Kt.reshape(-1, 3, 3)[:1].to(dev).contiguous()  # frame 0's camera (every frame's with K [3,3])
        self.K_frames = Kt.reshape(n_frames, 1, 3, 3).to(dev).contiguous() if Kt.dim() == 3 else None
        self.K_cur = self.Ks
        self.images, self.frames_kind, self.sizes = images, kind, sizes
        distinct = sorted(set(sizes))
        self.multi_size = len(distinct) > 1
        K_sh = (sh_degree + 1) ** 2
        net = sdf.net_mod
        cap = (int(capacity) + 3) // 4 * 4  # a multiple of 4 rows: every segment of the flat buffers starts 16-byte aligned
        T = self.T = RD.GsSdfTrainer(cap, K_sh, W, H, dev, int(isect_cap or 64 * cap), sdf.cfg, n_ray_samples=sdf.rs.cap,
                                     sh_degree=sh_degree, bce_sigma=sdf.bce_sigma, eikonal_weight=sdf.eik_w, gs_sdf_weight=gs_sdf_weight,
                                     visible_thr=visible_thr, mlp_mode=1, eikonal_mode=1, align_weight=sdf.align_w, rgb_weight=rgb_weight,
                                     dssim_weight=dssim_weight, depth_weight=0.0, normal_weight=0.0, isotropic_weight=isotropic_weight,
                                     spatial_scale=self.spatial_scale, n_live=n0, delta_dev=sdf.std_dev, bck_color=bck_color, mask=mask,
                                     depth_type=depth_type, frame_sizes=distinct if self.multi_size else None)
        T.origin, T.inv_size, T.bce_isigma = net.origin, net.inv_size, sdf.bce_isigma
        T.set_octree(sdf.rs.tree)
        n_sdf = sdf.n_table + sdf.n_mlp
        T.load(splats["anchors"], splats["offsets"], splats["quaternion"], splats["scaling"], splats["opacity"], splats["features_dc"],
               splats["features_rest"], sdf.table, sdf.mlp, sdf_exp_avg=sdf.exp_avg[:n_sdf], sdf_exp_avg_sq=sdf.exp_avg_sq[:n_sdf],
               sdf_step=sdf.t)
        if self.detach:  # freeze_net (:389-391): the SDF stage, the SDF callback and the SDF groups are off; [C] keeps its gs_sdf term only
            T.eik_w, T.align_w = 0.0, 0.0
        T.R.sh_degree = 0  # sh_degree_to_use_ = 0 at construction (neural_gaussian.cpp:406)
        dkw = dict(densify or {})
        dkw.update(sh_degree=sh_degree, sh_degree_interval=sh_degree_interval)
        self.D = DN.Densifier(T, n_frames, spatial_scale=self.spatial_scale, lr_end=sdf.lr_end, **dkw)
        self.D.pin_image_size = self.multi_size
        self.sdf_steps0 = sdf.t
        self.cpu_gen = torch.Generator().manual_seed(seed)
        self.gen = torch.Generator(dev).manual_seed(seed)
        self.bg_gen = torch.Generator(dev).manual_seed(seed + (1 << 32))  # bck_color 2's backgrounds: not the randns stream
        self.randns = torch.empty(T.R.cap, 2, dtype=torch.float32, device=dev)  # the splat samples' draw, fresh every render
        self.perm = None
        # RGB + the (unused) depth channel the loss kernels read, viewed at the current frame's size
        self._gt_store = torch.zeros(4 * T.R.max_pixels, dtype=torch.float32, device=dev)
        self.gt = self._gt_store[:4 * H * W].view(1, H, W, 4)
        pinned = [t for t in (images if kind == "list" else [store]) if not t.is_cuda]
        # staging for pinned frames: one frame's floats, or one frame's bytes of an 8-bit store
        self._stage_store = (None if not pinned else torch.empty(3 * T.R.max_pixels, dtype=torch.uint8 if kind == "u8" else torch.float32,
                                                                  device=dev))
        self.stage = self._stage_store[:3 * H * W].view(H, W, 3) if self._stage_store is not None and kind != "u8" else None
        f32, i32 = dict(dtype=torch.float32, device=dev), dict(dtype=torch.int32, device=dev)
        n_it = self.iters
        self.h_color = torch.zeros(n_frames if self.color_init else 0, **f32)
        self.h_loss, self.h_sdf_loss, self.h_std = torch.zeros(n_it, **f32), torch.zeros(n_it, **f32), torch.zeros(n_it, **f32)
        self.h_samples, self.h_vis = torch.zeros(n_it, **i32), torch.zeros(n_it, **i32)
        self.n_live_log = []  # host: live splats after each joint iteration
        self.done = 0

    # ---- pieces of one iteration --------------------------------------------------------------------------------------------------
    def camera(self, i):
        """train_cameras_idx[i % train_num], redrawn whenever i % train_num == 0 (the static tensor carries over from colour init)."""
        if perm_due(i, self.train_num) or self.perm is None:
            self.perm = torch.randperm(self.train_num, generator=self.cpu_gen).tolist()
        return self.perm[i % self.train_num]

    def set_frame(self, W, H):
        """Train at W x H from here on: the renderer, the background and the ground truth become views of that size."""
        if (self.T.R.W, self.T.R.H) == (W, H) and tuple(self.gt.shape[1:3]) == (H, W):
            return
        self.T.set_frame(W, H)
        self.gt = self._gt_store[:4 * H * W].view(1, H, W, 4)
        if self._stage_store is not None and self.frames_kind != "u8":
            self.stage = self._stage_store[:3 * H * W].view(H, W, 3)

    def load_frame(self, cam):
        """gt <- images[cam] (the reference's get_image(..).to(k_device)) at the frame's size, with the frame's K in K_cur; a pinned frame
        goes through the staging buffer asynchronously, an 8-bit frame is expanded on the device."""
        W, H = self.sizes[cam]
        self.set_frame(W, H)
        self.K_cur = self.Ks if self.K_frames is None else self.K_frames[cam]
        if self.frames_kind == "u8":
            st = self.images
            if st.is_cuda:
                cabi.frames_u8_expand(st.data, st.offsets[cam], W, H, self.gt)
            else:
                stage = self._stage_store[:3 * W * H]
                stage.copy_(st.data[st.offsets[cam]:st.offsets[cam + 1]], non_blocking=True)
                cabi.frames_u8_expand(stage, 0, W, H, self.gt)
        elif self.images[cam].is_cuda:
            self.gt[0, ..., :3].copy_(self.images[cam])
        else:
            self.stage.copy_(self.images[cam], non_blocking=True)
            self.gt[0, ..., :3].copy_(self.stage)
        return self.viewmats[cam:cam + 1]

    def draw_background(self):
        """bck_color 2: a fresh uniform background for the next render (torch::rand({H,W,3}), neural_gaussian.cpp:545-547)."""
        if self.T.bg is not None:
            self.T.bg.uniform_(generator=self.bg_gen)

    def run_color_init(self):
        """gs_train's color_init block (:364-387): train_num iterations of gs_train_batch_iter(i, false) + Adam over the SH groups."""
        T = self.T
        base = list(T.lr)
        T.lr = [10 * lr for lr in base]
        T.set_live(T.N_live)
        for i in range(self.train_num):
            vm = self.load_frame(self.camera(i))
            self.draw_background()
            T.color_step(vm, self.K_cur, self.gt)
            self.h_color[i:i + 1].copy_(T.R.loss)
        T.lr = [color_init_lr(lr) for lr in base]
        T.flat_grad[:T.t0].zero_()  # the structure's gradients of the frozen iterations are discarded
        T.set_live(T.N_live)

    def start_rates(self):
        """train_callback(0, k_gs_iter_step, p_optimizer_, empty_map): the rate decay alone (:392-394, neural_gaussian.cpp:604-623)."""
        T = self.T
        T.lr[0] = xyz_lr(0, self.iters, self.spatial_scale)
        T.sdf_lr = min(T.lr[0], self.D.lr_end)
        T.set_live(T.N_live)

    def step(self, i):
        """Joint iteration i, in the reference's order (:396-523)."""
        T, S, rs = self.T, self.sdf, self.sdf.rs
        vm = self.load_frame(self.camera(i))
        T.normal_w = self.normal_w if normal_on(i, self.refine_struct_start) else 0.0
        self.randns.normal_(generator=self.gen)  # the reference's randn of every render (Projection.cpp:728)
        self.draw_background()
        if self.detach:
            loss, sdf_loss = T.train_step(vm, self.K_cur, self.gt, None, None, self.randns)
        else:
            S.draw()
            cabi.sdf_ray_batch(S.pack, S.rand, S.n_rays_dev, S.rays)
            rs.sample(S.rays["origin"], S.rays["direction"], S.rays["depth"], S.rays["xyz"], n_live=S.n_rays_dev, sample_std=S.std_dev)
            torch.bitwise_or(S.overflow, rs.counts[2:3], out=S.overflow)
            loss, sdf_loss = T.train_step(vm, self.K_cur, self.gt, rs.xyz, rs.ray_sdf, self.randns, ray_n_live=rs.counts)
        T.adam_clocks(sdf=not self.detach)
        if self.detach:
            T.flat_grad[T.t0:].zero_()  # [C]'s SDF gradient has no optimiser group to consume it
        self.h_loss[i:i + 1].copy_(loss)
        self.h_sdf_loss[i:i + 1].copy_(sdf_loss)
        self.h_vis[i:i + 1].copy_(T.n_gate)
        if not self.detach:  # sdf_train_callback(i, k_gs_iter_step, point_samples, false) (:480-482, :533-593)
            cabi.sdf_adapt(S.adapt, T.ray_y1[:rs.cap], rs.counts, S.bce_sigma, S.bce_isigma, S.batch_pt_num, update_rays=False)
            self.h_samples[i:i + 1].copy_(rs.counts[0:1])
            if self.outlier_remove and outlier_due(i, self.outlier_interval):
                S.remove_outliers(i, total_iter=self.iters, net=T.sdf_net(), outlier_dist=self.outlier_dist)
        self.h_std[i:i + 1].copy_(S.std_dev)
        if callback_due(i, self.iters):  # NeuralGS::train_callback (:485-487) up to its early return
            T.R.sh_degree = self.D.train_callback(i, self.iters)
        self.n_live_log.append(T.N_live)
        self.done = i + 1

    def run(self):
        if self.color_init:
            self.run_color_init()
        self.start_rates()
        for i in range(self.iters):
            self.step(i)

    # ---- results ------------------------------------------------------------------------------------------------------------------
    def histories(self):
        """Per joint iteration: photometric loss, SDF loss, sample std after the iteration's update, sampler sample count, gated splat-sample
        count (vis_n); the colour-initialisation losses; and the host records of live splats and densification events. The device records
        (and the sampler's overflow flag) come back in one copy. Raises if the ray sampler's capacity overflowed."""
        n, nc = self.done, self.h_color.numel()
        f = lambda t: t.view(torch.float32) if t.dtype == torch.int32 else t
        parts = [self.sdf.overflow, self.h_loss[:n], self.h_sdf_loss[:n], self.h_std[:n], self.h_samples[:n], self.h_vis[:n], self.h_color]
        host = torch.cat([f(t) for t in parts]).cpu().numpy()
        if int(host[:1].view(np.int32)[0]):
            raise RuntimeError("GsTrainer: the ray sampler's sample or nugget capacity overflowed")
        r = [host[1 + k * n:1 + (k + 1) * n] for k in range(5)]
        return dict(loss=r[0], sdf_loss=r[1], sample_std=r[2], n_samples=r[3].view(np.int32), vis_n=r[4].view(np.int32),
                    color_loss=host[1 + 5 * n:1 + 5 * n + nc], n_live=np.asarray(self.n_live_log, np.int64), densify_events=list(self.D.log))

    def state(self):
        """dict(net=the SdfNet with the trained SDF written back (mesh.meshing), splats=the trained splats as io.export_gs_to_ply takes them
        (anchors, offsets, features_dc, features_rest, opacity, scaling, quaternion), render(viewmat, camera=None) -> [H,W,3] image for
        metrics.eval_render)."""
        T = self.T
        p = T.params  # brings every SH row current
        with torch.no_grad():
            self.sdf.net_mod.params_.copy_(T.table)
            self.sdf.net_mod.decoder_.copy_(T.mlp)
        sc = T.scene
        splats = dict(anchors=T.anchors, offsets=sc["raw"]["offsets"], features_dc=sc["sh"],
                      features_rest=sc["raw"]["sh_rest"] if sc["raw"]["sh_rest"] is not None else p.new_zeros(T.N_live, 0, 3),
                      opacity=sc["opacities"], scaling=sc["scales"], quaternion=sc["quats"])
        return dict(net=self.sdf.net_mod, splats=splats, render=self.render)

    def render(self, viewmat, camera=None):
        """The colour image [H,W,3] of a world->camera pose [4,4] at the current SH degree on the configured background (the render the
        reference exports and scores; bck_color 2 draws a fresh background for it). camera: (W, H, K [3,3]), e.g. an entry of
        io.load_colmap_cameras' table; None renders with frame 0's camera. Its pixel count and tile grid must fit the largest training
        frame's (the renderer's storage)."""
        T = self.T
        T.flush_sh()
        vm = torch.as_tensor(viewmat, dtype=torch.float32).reshape(1, 4, 4).to(self.dev).contiguous()
        if camera is None:
            (W, H), K = self.sizes[0], self.Ks
        else:
            W, H, K = int(camera[0]), int(camera[1]), torch.as_tensor(camera[2], dtype=torch.float32).reshape(1, 3, 3).to(self.dev).contiguous()
        T.view_frame(W, H)  # the image mask belongs to the loss, not to the render
        sc = T.scene
        raw = dict(sc["raw"], sh_catch_up=None)
        self.draw_background()
        T.R.forward(sc["means"], sc["quats"], sc["scales"], sc["opacities"], sc["sh"], vm, K, raw=raw, bck_color=T.bck_color, bg=T.bg)
        return T.R.out_colors[0, ..., :3].clone()

    def __repr__(self):
        return f"GsTrainer(N_live={self.T.N_live}, capacity={self.T.N_cap}, frames={self.train_num}, iters={self.iters})"
