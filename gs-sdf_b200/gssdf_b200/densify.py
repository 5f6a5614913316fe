"""Host mirror of NeuralGS's densification strategy (include/neural_gaussian/neural_gaussian.cpp:568-926: train_callback, update_state,
grow_gs / duplicate / split, prune_gs, prune_invisible_gs, prune_nan_gs, reset_opacity, learning-rate decay) over the densify kernels of
the C ABI, acting on a render.GsSdfTrainer (flat parameter / Adam-moment buffers with a row capacity).

The per-iteration part (`update_state`) is asynchronous. A refinement event reads the decision flags back once (the reference calls
.sum().item() / nonzero() a dozen times per event) and rebuilds parameters + moments with one remap kernel per surgery step. Under data
parallelism call `parallel.allreduce_densify_state(D.state)` before `train_callback` and give every rank the same `generator` seed: the
decisions and the split noise are then identical on every replica (SURVEY 8e)."""
import math

import torch

from . import cabi

DUPLI, SPLIT, P_OPA, P_SMALL, P_BIG, P_NAN, P_INVIS = 1, 2, 4, 8, 16, 32, 64


class Densifier:
    def __init__(self, trainer, num_train_data, spatial_scale=1.0, sh_degree=3, prune_opa=0.05, grow_grad2d=0.0002, grow_scale3d=0.01,
                 grow_scale2d=0.05, prune_scale3d=0.1, refine_scale2d_stop_iter=0, refine_start_iter=500, refine_every=100,
                 reset_alpha_every=30, sh_degree_interval=1000, lr_end=1e-4, pause_refine_after_reset=None, generator=None):
        """Defaults = config/base.yaml:62-76 (prune_opa .. sh_degree_interval)."""
        T = self.T = trainer
        self.dev, self.N_cap = T.dev, T.N_cap
        z = lambda: torch.zeros(self.N_cap, dtype=torch.float32, device=self.dev)
        self.state = dict(grad2d=z(), count=z(), vis=z(), radii=z())
        self.state2 = {k: torch.zeros_like(v) for k, v in self.state.items()}
        self.flags = torch.zeros(self.N_cap, dtype=torch.uint8, device=self.dev)
        self.alt = None  # second set of flat buffers for the remap (allocated at the first surgery)
        self.num_train_data, self.spatial_scale, self.orig_spatial_scale = num_train_data, spatial_scale, spatial_scale
        self.k_sh_degree, self.sh_degree_interval = sh_degree, sh_degree_interval
        self.prune_opa, self.grow_grad2d, self.grow_scale3d, self.grow_scale2d = prune_opa, grow_grad2d, grow_scale3d, grow_scale2d
        self.prune_scale3d, self.scale2d_stop, self.refine_start, self.refine_every = prune_scale3d, refine_scale2d_stop_iter, refine_start_iter, refine_every
        self.reset_every = reset_alpha_every * refine_every  # params.cpp:429
        # neural_gaussian.cpp:286-290: _num_train_data when the scene is large, else 0
        self.pause_after_reset = num_train_data if pause_refine_after_reset is None else pause_refine_after_reset
        self.lr_end = lr_end
        self.gen = generator or torch.Generator(self.dev).manual_seed(0)
        self.log = []
        # frames of several sizes (gstrain.GsTrainer with a camera per frame): the radii normaliser is max(W, H) of the first update,
        # as the reference's `static image_size` (:658); grad2d keeps each frame's own scaling. False: every update normalises by its own
        # frame, which is the same value when there is one size.
        self.pin_image_size = False
        self.image_size = None

    # ---- every iteration --------------------------------------------------------------------------------------------------------
    def update_state(self):
        """NeuralGS::update_state (:626-680) from the renderer's buffers of the step that just ran; no host sync."""
        R = self.T.R
        if self.pin_image_size and self.image_size is None:
            self.image_size = float(max(R.W, R.H))
        cabi.densify_update_state(self.T.N_live, R.cap, R.counts, R.p["gaussian_ids"], R.g["v_densify"], R.r["visibilities"],
                                  R.p["radii"] if self.scale2d_stop > 0 else None, R.W, R.H, R.C, self.state["grad2d"], self.state["count"],
                                  self.state["vis"], self.state["radii"] if self.scale2d_stop > 0 else None,
                                  image_size=self.image_size if self.pin_image_size else None)

    # ---- surgery ----------------------------------------------------------------------------------------------------------------
    def _flags(self, with_grow, it):
        T, n = self.T, self.T.N_live
        sc = T.scene
        cabi.densify_flags(n, sc["raw"]["offsets"], sc["quats"], sc["scales"], sc["opacities"], self.flags,
                           grad2d=self.state["grad2d"] if with_grow else None, count=self.state["count"] if with_grow else None,
                           vis=self.state["vis"], radii_state=self.state["radii"], grow_grad2d=self.grow_grad2d,
                           grow_scale3d=self.grow_scale3d * self.spatial_scale, grow_scale2d=self.grow_scale2d,
                           use_scale2d=it < self.scale2d_stop, prune_opa=self.prune_opa, prune_scale3d=self.prune_scale3d * self.orig_spatial_scale)
        return self.flags[:n]

    def _remap(self, src, mode, randn_row=None, randn=None):
        """Rebuild the trainer's splat rows: new row r <- old row src[r] under `mode` (0 keep, 1 duplicate, 2 split sample)."""
        T = self.T
        n_new = int(src.numel())
        if n_new > T.N_cap:
            raise RuntimeError(f"densification needs {n_new} rows but the trainer was built with a capacity of {T.N_cap}")
        if self.alt is None:
            self.alt = dict(params=torch.zeros_like(T.params), exp_avg=torch.zeros_like(T.exp_avg), exp_avg_sq=torch.zeros_like(T.exp_avg_sq),
                            anchors=torch.zeros_like(T.anchors_buf))
        old = dict(params=T.params, exp_avg=T.exp_avg, exp_avg_sq=T.exp_avg_sq, anchors=T.anchors_buf)
        names = ["grad2d", "count", "vis", "radii"]
        cabi.densify_remap(n_new, T.R.K, T.N_cap, T.N_cap, src.to(torch.int32).contiguous(), mode.to(torch.uint8).contiguous(),
                           randn_row.to(torch.int32).contiguous() if randn_row is not None else None, randn, old, self.alt,
                           [self.state[k] for k in names], [self.state2[k] for k in names])
        t0 = T.t0
        for k in ("params", "exp_avg", "exp_avg_sq"):  # the SDF segment (hash table + decoder) travels with the buffer swap
            self.alt[k][t0:].copy_(old[k][t0:])
        T.params, T.exp_avg, T.exp_avg_sq, T.anchors_buf = self.alt["params"], self.alt["exp_avg"], self.alt["exp_avg_sq"], self.alt["anchors"]
        T.stamp_sh_current()  # reading T.params above brought every SH row current: the remapped rows are copies of current rows
        self.alt = old
        self.state, self.state2 = self.state2, self.state
        T.set_live(n_new)
        T.flat_grad[:t0].zero_()  # gradients of the old row numbering are meaningless now

    def grow_gs(self, it):
        """grow_gs (:690-720) = duplicate (:722-760) then split (:762-826): rows [non-split rows in order | duplicates | split k=0 | split k=1]."""
        f = self._flags(True, it)
        n = self.T.N_live
        dupli_idx = torch.nonzero(f & DUPLI).flatten()
        is_split = torch.cat([(f & SPLIT) != 0, torch.zeros(dupli_idx.numel(), dtype=torch.bool, device=self.dev)])
        src1 = torch.cat([torch.arange(n, device=self.dev), dupli_idx])
        mode1 = torch.cat([torch.zeros(n, dtype=torch.uint8, device=self.dev), torch.ones(dupli_idx.numel(), dtype=torch.uint8, device=self.dev)])
        sel, rest = torch.nonzero(is_split).flatten(), torch.nonzero(~is_split).flatten()
        ns, K = int(sel.numel()), 2
        src = torch.cat([src1[rest]] + [src1[sel]] * K)
        mode = torch.cat([mode1[rest], torch.full((K * ns,), 2, dtype=torch.uint8, device=self.dev)])
        randn = torch.randn(K, ns, 3, device=self.dev, generator=self.gen).reshape(-1, 3).contiguous() if ns else None  # torch::randn({K, n_split, 3})
        randn_row = torch.cat([torch.zeros(rest.numel(), dtype=torch.int32, device=self.dev), torch.arange(K * ns, dtype=torch.int32, device=self.dev)])
        if dupli_idx.numel() or ns:
            self._remap(src, mode, randn_row, randn)
        return int(dupli_idx.numel()), ns

    def _prune(self, is_prune):
        n_prune = int(is_prune.sum())
        if n_prune > 0:
            valid = torch.nonzero(~is_prune).flatten()
            self._remap(valid, torch.zeros(valid.numel(), dtype=torch.uint8, device=self.dev))
        return n_prune

    def prune_gs(self, it, prune_opa_only=False):
        f = self._flags(False, it)
        m = P_OPA | P_SMALL | (P_BIG if (not prune_opa_only and it > self.reset_every) else 0)
        return self._prune((f & m) != 0)

    def prune_invisible_gs(self, it):
        if it > 0 and it % self.num_train_data == 0:
            f = self._flags(False, it)
            is_prune = (f & P_INVIS) != 0
            self.state["vis"].zero_()
            return self._prune(is_prune)
        return 0

    def prune_nan_gs(self, it):
        return self._prune((self._flags(False, it) & P_NAN) != 0)

    def reset_opacity(self):
        """reset_opacity (:907-915): opacity_ = min(opacity_, logit(2 prune_opa)); the Adam moments of the opacity group are zeroed
        (replace_tensors_to_optimizer, optimizer_utils.cpp)."""
        T, n = self.T, self.T.N_live
        cap = math.log(2 * self.prune_opa / (1 - 2 * self.prune_opa))
        T.scene["opacities"].clamp_(max=cap)
        o = T.seg_off[3]
        T.exp_avg[o:o + n].zero_()
        T.exp_avg_sq[o:o + n].zero_()

    # ---- schedule ---------------------------------------------------------------------------------------------------------------
    def train_callback(self, it, total_iter):
        """NeuralGS::train_callback (:568-624). Returns the SH degree to use next (sh_degree_to_use_)."""
        T = self.T
        refine_stop = total_iter // 2
        if it < refine_stop:
            self.update_state()
            self.prune_nan_gs(it)
            self.prune_invisible_gs(it)
        sh = min(self.k_sh_degree, it // self.sh_degree_interval)
        if 0 < it < refine_stop:
            if it > self.refine_start and it % self.refine_every == 0 and (it % self.reset_every) >= self.pause_after_reset:
                nd, ns = self.grow_gs(it)
                npr = self.prune_gs(it)
                self.state["grad2d"].zero_(); self.state["count"].zero_()
                if self.scale2d_stop > 0:
                    self.state["radii"].zero_()
                self.log.append((it, nd, ns, npr, T.N_live))
            if it % self.reset_every == 0:
                self.reset_opacity()
        # learning-rate decay (:604-623)
        ratio = it / float(total_iter)
        lr0, lr1 = 1.6e-4 * self.spatial_scale, 1.6e-6 * self.spatial_scale
        xyz_lr = math.exp(math.log(lr0) * (1 - ratio) + math.log(lr1) * ratio)
        T.lr[0] = xyz_lr
        T.sdf_lr = min(xyz_lr, self.lr_end)
        T.set_live(T.N_live)
        return sh
