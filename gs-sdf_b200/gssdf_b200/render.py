"""Asynchronous, capacity-based render + backward of the splat path (the throughput path).

`SplatRenderer.step()` runs SURVEY.md section 3.2 [B]+[D] for one camera batch entirely through the C ABI
with ZERO host synchronisation: projection -> SH colour -> tile keys/sort/offsets -> rasterise ->
post-ops -> L1 loss + cotangents -> post-ops bwd -> rasterise bwd -> SH bwd -> projection bwd.
The visible-splat count and the intersection count live in a device-side `gssdf_counts`; buffers are
sized by capacity (cap = C*N rows, isect_cap chosen by the caller) and overflow is flagged there.
All gradients land in ONE flat fp32 buffer (means|quats|scales|opacities|sh) so that data-parallel
training is a single NCCL all-reduce (SURVEY 8e).
"""
import contextlib
import math

import torch

from . import cabi


def check_photometric(who, bck_color, mask, H, W, device):
    """The background mode and image mask of the photometric path (DESIGN 7o), checked before any device work: bck_color 0 (black),
    1 (white) or 2 (random); mask None or a bool / uint8 tensor [H,W], [H,W,1] or [H,W,3] on the CUDA device `device`."""
    if isinstance(bck_color, bool) or bck_color not in (0, 1, 2):
        raise ValueError(f"{who}: bck_color must be 0 (black), 1 (white) or 2 (random), got {bck_color!r}")
    if mask is None:
        return
    if not isinstance(mask, torch.Tensor) or mask.dtype not in (torch.bool, torch.uint8):
        raise ValueError(f"{who}: mask must be a bool or uint8 tensor, got {getattr(mask, 'dtype', type(mask))}")
    if H is not None and tuple(mask.shape) not in ((H, W), (H, W, 1), (H, W, 3)):
        raise ValueError(f"{who}: mask must be [H,W], [H,W,1] or [H,W,3] with H={H}, W={W}, got {tuple(mask.shape)}")
    dev = torch.device(device)
    if not mask.is_cuda or dev.type != "cuda" or (dev.index is not None and mask.device.index != dev.index):
        raise ValueError(f"{who}: mask must be on {dev}, got {mask.device}")


def check_depth_type(who, depth_type):
    """k_depth_type, the depth the normal-consistency term and the depth-to-normal frame differentiate (neural_mapping.cpp:248-252,
    config/base.yaml:43): 0 the expected depth, any other int the rasteriser's median depth (bounded scenes; the COLMAP configurations'
    `depth_type`). Returns True for the median."""
    if isinstance(depth_type, bool) or not isinstance(depth_type, int):
        raise ValueError(f"{who}: depth_type must be an int (0: expected depth, otherwise the median depth), got {depth_type!r}")
    return depth_type != 0


def expand_mask(mask, H, W):
    """A checked mask as the masked loss kernels read it: uint8 [H,W,3], nonzero -> 1 (the reference's bool mask)."""
    return None if mask is None else mask.reshape(H, W, -1).ne(0).to(torch.uint8).expand(H, W, 3).contiguous()


def frame_maxima(sizes, tile_size=16):
    """(largest pixel count, largest tile count) over a list of (W, H) frame sizes: what per-pixel and per-tile storage must hold."""
    return (max(int(w) * int(h) for w, h in sizes),
            max(math.ceil(int(w) / tile_size) * math.ceil(int(h) / tile_size) for w, h in sizes))


# per-pixel buffers of SplatRenderer: (dict attribute or None, key, channels, dtype, zero-initialised)
_PIXEL_BUFFERS = [("r", "render_colors", 3, torch.float32, False), ("r", "render_depths", 1, torch.float32, False),
                  ("r", "render_alphas", 1, torch.float32, False), ("r", "render_normals", 3, torch.float32, False),
                  ("r", "render_median", 1, torch.float32, False), ("r", "last_ids", None, torch.int32, False),
                  ("r", "median_ids", None, torch.int32, False), (None, "out_colors", 4, torch.float32, False),
                  (None, "out_normals", 3, torch.float32, False), (None, "v_out_colors", 4, torch.float32, False),
                  (None, "v_out_normals", 3, torch.float32, True), ("v_r", "colors", 3, torch.float32, False),
                  ("v_r", "depths", 1, torch.float32, False), ("v_r", "alphas", 1, torch.float32, False),
                  ("v_r", "normals", 3, torch.float32, False), ("v_r", "median", 1, torch.float32, True)]


class SplatRenderer:
    def __init__(self, N, K, C, W, H, device, isect_cap, tile_size=16, near=0.05, far=300.0, sh_degree=3, presort_cull=True,
                 frame_sizes=None):
        """frame_sizes: every (W, H) the renderer will be asked to render (DESIGN 7q). Per-pixel and per-tile storage is allocated for the
        largest pixel count and the largest tile grid among them and `set_frame` re-views it as contiguous [C,H,W,.] buffers of one
        size; the raster, tile and DSSIM workspaces are sized for the maxima. None: (W, H) only, today's exact allocation. The renderer
        starts at (W, H)."""
        self.N, self.K, self.C, self.tile = N, K, C, tile_size
        self.near, self.far, self.sh_degree = near, far, sh_degree
        self.dev = device
        self.cap = N * C
        self.isect_cap = int(isect_cap)
        self.frame_sizes = [(int(W), int(H))] + [(int(w), int(h)) for w, h in (frame_sizes or [])]
        self.max_pixels, self.max_tiles = frame_maxima(self.frame_sizes, tile_size)
        f32 = dict(dtype=torch.float32, device=device)
        i32 = dict(dtype=torch.int32, device=device)
        cap = self.cap
        e = lambda *s, **k: torch.empty(*s, **(k or f32))
        self.counts = torch.zeros(cabi.COUNTS_INTS, **i32)
        self.p = dict(camera_ids=e(cap, dtype=torch.int64, device=device), gaussian_ids=e(cap, dtype=torch.int64, device=device),
                      radii=e(cap, 2, **i32), means2d=e(cap, 2), depths=e(cap), ray_transforms=e(cap, 3, 3), normals=e(cap, 3),
                      samples=e(cap, 3), sample_weights=e(cap, 1), pt_opacities=e(cap), indptr=e(C + 1, **i32))
        self.colors = e(cap, 3)
        self.presort_cull = bool(presort_cull) and tile_size == 16
        self.conics = e(cap, 8) if self.presort_cull else None
        self.flatten_ids = e(self.isect_cap, **i32)
        # flat storage behind every per-pixel buffer and the tile offsets; set_frame views its leading C*H*W*channels elements.
        # no render_distort / render_Ts: the distortion loss is off in GS-SDF (distloss = false), the kernel then skips those terms
        self._pix = {}
        for grp, key, ch, dt, zero in _PIXEL_BUFFERS:
            n = C * self.max_pixels * (ch or 1)
            self._pix[(grp, key)] = (torch.zeros if zero else torch.empty)(n, dtype=dt, device=device)
        self._offsets_store = e(C * self.max_tiles, **i32)
        self.r, self.v_r = {}, {}
        self.W = self.H = None
        self.set_frame(W, H)
        self.r["visibilities"] = e(cap, 1)
        self.g = dict(v_means2d=None, v_ray_transforms=e(cap, 3, 3), v_colors=e(cap, 3), v_opacities=e(cap),
                      v_normals=e(cap, 3), v_densify=e(cap, 2))
        # flat gradient buffer: means[N,3] quats[N,4] scales[N,3] opacities[N] sh[N,K,3]
        sizes = [N * 3, N * 4, N * 3, N, N * K * 3]
        self.flat_grad = torch.zeros(sum(sizes), **f32)
        o = [0]
        for s in sizes:
            o.append(o[-1] + s)
        fg = self.flat_grad
        self.v_means, self.v_quats = fg[o[0]:o[1]].view(N, 3), fg[o[1]:o[2]].view(N, 4)
        self.v_scales, self.v_opac, self.v_sh = fg[o[2]:o[3]].view(N, 3), fg[o[3]:o[4]], fg[o[4]:o[5]].view(N, K, 3)
        self.loss = torch.zeros(1, **f32)
        self.ws = cabi.Workspace(device)
        # dedicated raster workspace (records, conics, culled lists | gradient records): the backward reuses the forward's part
        self.raster_ws = cabi.Workspace(device)
        self.loss_ws = cabi.Workspace(device)  # DSSIM derivative maps
        L, i64 = cabi.lib(), cabi._lib.C.c_int64
        self.raster_ws.get(max(L.gssdf_raster2dgs_bwd_workspace_bytes(C, w, h, cap, i64(self.isect_cap)) for w, h in self.frame_sizes))
        if frame_sizes:  # several sizes: no workspace grows between frames
            self.ws.get(max(max(L.gssdf_tile_encode_workspace_bytes(C, w, h, tile_size, i64(self.isect_cap)),
                                L.gssdf_project2dgs_workspace_bytes(N, C)) for w, h in self.frame_sizes))
            self.loss_ws.get(max(L.gssdf_dssim_workspace_bytes(C, w, h) for w, h in self.frame_sizes))
        self.prof_fwd = self.prof_bwd = None  # optional (start, stop) torch.cuda.Event pairs around the raster kernels
        self.stage_events = None  # profiling: list of (stage name, torch.cuda.Event recorded AFTER the stage) (bench.py per-stage table)

    def set_frame(self, W, H):
        """Render frames of W x H from here on: every per-pixel buffer (r, v_r, out_*, v_out_*) and the tile offsets become contiguous
        [C,H,W,.] views of the leading elements of their storage. The size must fit the storage frame_sizes allocated; the pixels past a
        smaller frame keep whatever a larger one left there, and no kernel reads them."""
        W, H = int(W), int(H)
        if (W, H) == (self.W, self.H):
            return
        tw, th = math.ceil(W / self.tile), math.ceil(H / self.tile)
        if W < 1 or H < 1 or W * H > self.max_pixels or tw * th > self.max_tiles:
            raise ValueError(f"SplatRenderer.set_frame: a {W}x{H} frame does not fit storage for {self.max_pixels} pixels and "
                             f"{self.max_tiles} tiles (frame_sizes)")
        C = self.C
        self.W, self.H, self.tw, self.th = W, H, tw, th
        for grp, key, ch, _, _ in _PIXEL_BUFFERS:
            st = self._pix[(grp, key)]
            v = st[:C * H * W * (ch or 1)].view((C, H, W, ch) if ch else (C, H, W))
            if grp is None:
                setattr(self, key, v)
            else:
                getattr(self, grp)[key] = v
        self.offsets = self._offsets_store[:C * th * tw].view(C, th, tw)

    def _zero_pixels(self, grp, key):
        """Zero a buffer's whole storage (the tail a smaller frame does not view included)."""
        self._pix[(grp, key)].zero_()

    def _mark(self, name):
        if self.stage_events is not None:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            self.stage_events.append((name, ev))

    # -- forward ------------------------------------------------------------------------------
    def forward(self, means, quats, scales, opacities, sh, viewmats, Ks, randns=None, raw=None, bck_color=0, bg=None):
        """raw = dict(offsets=[N,3], sh_rest=[N,K-1,3]) switches to the RAW parameters of NeuralGS (row a1 fused into the kernels):
        means = anchors, scales = log-scales, opacities = logits, sh = features_dc; no activated copies are materialised.
        bck_color: the background composited into out_colors after the rasteriser (NeuralGS::render): 0 black, 1 white, 2 the image
        bg [C,H,W,3]."""
        C, W, H, cap = self.C, self.W, self.H, self.cap
        off, rest = (raw["offsets"], raw["sh_rest"]) if raw else (None, None)
        cabi.project2dgs_fwd(means, quats, scales, viewmats, Ks, W, H, self.near, self.far, 0.0, randns, cap, self.p,
                             self.counts, self.ws, opacities=opacities, mean_offsets=off, raw_params=raw is not None)
        self._mark("projection_fwd")
        if raw and raw.get("sh_catch_up") is not None:  # lazy Adam (GsSdfTrainer): the visible SH rows are brought current first
            raw["sh_catch_up"]()
        cabi.view_colors_fwd(viewmats, means, sh, self.sh_degree, cap, self.counts, self.p["camera_ids"],
                             self.p["gaussian_ids"], self.p["radii"], self.colors, mean_offsets=off, sh_rest=rest)
        self._mark("sh_fwd")
        conics = None
        if self.presort_cull:  # exact footprint test BEFORE the sort: ~4x fewer keys to scatter / sort / cull
            cabi.splat_conics(cap, W, H, self.counts, self.p["ray_transforms"], self.p["pt_opacities"], self.conics)
            conics = self.conics
        cabi.tile_encode(C, W, H, self.tile, cap, self.counts, self.p["means2d"], self.p["radii"], self.p["depths"],
                         self.p["camera_ids"], self.isect_cap, None, None, self.flatten_ids, self.offsets, self.ws, conics=conics)
        self._mark("tile_encode")
        cabi.raster2dgs_fwd(C, W, H, self.tile, 3, cap, self.counts, self.p["means2d"], self.p["ray_transforms"], self.colors,
                            self.p["pt_opacities"], self.p["normals"], None, self.offsets, self.flatten_ids, self.r, self.raster_ws,
                            prof=self.prof_fwd, isect_cap=self.isect_cap)
        self._mark("raster_fwd")
        if bck_color:
            cabi.render_post_bg_fwd(C, W, H, viewmats, self.r["render_colors"], self.r["render_depths"], self.r["render_alphas"],
                                    self.r["render_normals"], self.out_colors, self.out_normals, bck_color, bg)
        else:
            cabi.render_post_fwd(C, W, H, viewmats, self.r["render_colors"], self.r["render_depths"], self.r["render_alphas"],
                                 self.r["render_normals"], self.out_colors, self.out_normals)
        self._mark("post_fwd")
        return self.out_colors, self.out_normals

    # -- loss + backward -----------------------------------------------------------------------
    def backward(self, means, quats, scales, opacities, sh, viewmats, Ks, gt, randns=None, w_rgb=1.0, w_depth=0.1, v_samples=None,
                 zero_grads=True, raw=None, w_dssim=0.0, w_normal=0.0, w_isotropic=0.0, before_projection_bwd=None, projection_bwd=True,
                 bck_color=0, bg=None, mask=None, median_depth=False):
        """With raw parameters the flat gradient holds dL/d(offsets|quats|log-scales|logits|features_dc|features_rest); the SH segment
        keeps its [N,K,3] size, laid out as dc [N,1,3] followed by rest [N,K-1,3]. projection_bwd=False stops after the SH backward (the
        structure is frozen: only the colour gradient is wanted). bck_color / bg: those of the forward; mask: uint8 [H,W,3]
        (expand_mask) multiplying both images in the L1 and DSSIM terms (loss::rgb_loss / dssim_loss with a mask). median_depth: the
        normal term differentiates render_median instead of the expected depth (check_depth_type); its depth cotangent then enters the
        rasteriser backward as v_render_median."""
        C, W, H, cap = self.C, self.W, self.H, self.cap
        off, rest = (raw["offsets"], raw["sh_rest"]) if raw else (None, None)
        N, K = self.N, self.K
        v_sh, v_rest = ((self.v_sh.view(-1)[:N * 3].view(N, 1, 3), self.v_sh.view(-1)[N * 3:].view(N, K - 1, 3)) if rest is not None
                        else (self.v_sh, None))
        self.loss.zero_()
        if zero_grads:
            self.flat_grad.zero_()
        if mask is None:
            cabi.l1_loss(C, W, H, self.out_colors, gt, w_rgb, w_depth, self.loss, self.v_out_colors)
        else:
            cabi.l1_loss_masked(C, W, H, self.out_colors, gt, w_rgb, w_depth, self.loss, self.v_out_colors, mask)
        if w_dssim > 0:  # + w_dssim * (1 - SSIM(rgb, gt)) (loss::dssim_loss), gradient added to the colour cotangent
            if mask is None:
                cabi.dssim_loss(C, W, H, self.out_colors, gt, w_dssim, self.loss, self.v_out_colors, self.loss_ws)
            else:
                cabi.dssim_loss_masked(C, W, H, self.out_colors, gt, w_dssim, self.loss, self.v_out_colors, self.loss_ws, mask)
        if w_normal > 0 and median_depth:  # the same term on the median depth (k_depth_type != 0): the kernel adds to v_render_median,
                                           # which is zero outside this branch
            self.v_r["median"].zero_()
            cabi.normal_consistency_loss(C, W, H, viewmats, Ks, self.r["render_median"], 1, self.r["render_alphas"], self.out_normals,
                                         w_normal, self.loss, v_depth=self.v_r["median"], v_depth_stride=1, v_out_normals=self.v_out_normals)
            self._v_normals_dirty = self._v_median_dirty = True
        elif w_normal > 0:  # normal consistency between the rendered normals and the normals of the expected-depth map
                            # (neural_mapping.cpp:243-266): adds to the ED cotangent (channel 3) and overwrites the normal cotangent
            cabi.normal_consistency_loss(C, W, H, viewmats, Ks, self.out_colors.data_ptr() + 12, 4, self.r["render_alphas"], self.out_normals,
                                         w_normal, self.loss, v_depth=self.v_out_colors.data_ptr() + 12, v_depth_stride=4,
                                         v_out_normals=self.v_out_normals)
            self._v_normals_dirty = True
        elif getattr(self, "_v_normals_dirty", False):  # the whole storage: a later, larger frame must read zeros too
            self._zero_pixels(None, "v_out_normals")
            self._v_normals_dirty = False
        if not (w_normal > 0 and median_depth) and getattr(self, "_v_median_dirty", False):
            self._zero_pixels("v_r", "median")
            self._v_median_dirty = False
        if w_isotropic > 0:  # isotropic regulariser on the visible splats' (x, y) scales (neural_mapping.cpp:268-276)
            cabi.isotropic_loss(self.N, cap, self.counts, self.p["gaussian_ids"], scales, raw is not None, w_isotropic, self.loss,
                                self.v_scales)
        if bck_color:
            cabi.render_post_bg_bwd(C, W, H, viewmats, self.r["render_depths"], self.r["render_alphas"], self.v_out_colors,
                                    self.v_out_normals, None, self.v_r["colors"], self.v_r["depths"], self.v_r["alphas"],
                                    self.v_r["normals"], bck_color, bg)
        else:
            cabi.render_post_bwd(C, W, H, viewmats, self.r["render_depths"], self.r["render_alphas"], self.v_out_colors,
                                 self.v_out_normals, None, self.v_r["colors"], self.v_r["depths"], self.v_r["alphas"],
                                 self.v_r["normals"])
        self._mark("losses+post_bwd")
        cabi.raster2dgs_bwd(C, W, H, self.tile, 3, cap, self.counts, self.p["means2d"], self.p["ray_transforms"], self.colors,
                            self.p["pt_opacities"], self.p["normals"], None, self.offsets, self.flatten_ids,
                            self.r["render_alphas"], None, self.r["last_ids"], self.r["median_ids"],
                            self.v_r["colors"], self.v_r["depths"], self.v_r["alphas"], self.v_r["normals"],
                            self.v_r["median"], self.g, self.raster_ws, prof=self.prof_bwd, isect_cap=self.isect_cap, reuse_fwd=True)
        self._mark("raster_bwd")
        cabi.view_colors_bwd(viewmats, means, sh, self.sh_degree, cap, self.counts, self.p["camera_ids"],
                             self.p["gaussian_ids"], self.p["radii"], self.colors, self.g["v_colors"], v_sh, self.v_means,
                             mean_offsets=off, sh_rest=rest, v_sh_rest=v_rest)
        self._mark("sh_bwd")
        if not projection_bwd:
            return self.loss
        if before_projection_bwd is not None:  # v_samples may be produced on another stream (GsSdfStep.overlap)
            before_projection_bwd()
        cabi.project2dgs_bwd(means, quats, scales, viewmats, Ks, W, H, cap, self.counts, self.p["camera_ids"],
                             self.p["gaussian_ids"], self.p["ray_transforms"], randns, None, None, self.g["v_ray_transforms"],
                             self.g["v_normals"], v_samples, self.v_means, self.v_quats, self.v_scales,
                             v_pt_opacities=self.g["v_opacities"], v_opacities=self.v_opac, mean_offsets=off,
                             raw_params=raw is not None, pt_opacities=self.p["pt_opacities"])
        self._mark("projection_bwd")
        return self.loss

    def step(self, scene, viewmats, Ks, gt, randns=None):
        raw = scene.get("raw")
        self.forward(scene["means"], scene["quats"], scene["scales"], scene["opacities"], scene["sh"], viewmats, Ks, randns, raw=raw)
        return self.backward(scene["means"], scene["quats"], scene["scales"], scene["opacities"], scene["sh"], viewmats, Ks, gt,
                             randns, raw=raw)

    # kernels launched by one step() (fwd: 3+1+6+2+1, bwd: 1+1+3+1+1 ; memsets not counted)
    KERNELS_PER_STEP = 21

    def read_counts(self):
        c = self.counts.cpu().tolist()
        return dict(nnz=c[0], n_isects=c[1], nnz_overflow=c[2], isect_overflow=c[3], max_tile_count=c[4], n_isects_aabb=c[6])


class GsSdfStep:
    """One full GS-SDF hot-path step (SURVEY.md section 3.2 [A]-[D]) with zero host synchronisation:

      [A] SDF on ray samples   : get_sdf(x) + 6-offset numerical gradient -> BCE + eikonal -> backward to table / decoder
      [B] render               : SplatRenderer.forward (projection -> SH -> tiles -> raster -> post-ops)
      [C] GS<->SDF coupling    : get_sdf(splat samples) (+ numerical eikonal) -> 0.5 sum w sdf^2, w = sample_weight * visibility
                                 (vis > visible_thr); its gradient w.r.t. the samples flows into the projection backward
      [D] backward             : L1 photometric/depth loss -> raster bwd -> SH bwd -> projection bwd
    All gradients land in ONE flat buffer [splat grads | table grad | decoder grad] (single all-reduce under data parallelism).
    eikonal_mode 1 (default with the tensor-core decoder): eikonal + align on the ANALYTIC gradient with the tcnn double backward, the
    reference default (config/base.yaml:13); eikonal_mode 0: the 6-offset numerical-gradient branch (local_map.cpp:110-133).
    Stage [C] applies the reference's sample gate (vis > visible_thr [& octree validity]): eikonal / align / coupling act on the gated
    samples only and their means divide by the gated count (neural_mapping.cpp:428-452).
    """

    def __init__(self, N, K, W, H, device, isect_cap, sdf_net_cfg, n_ray_samples=32768, sh_degree=3, origin=(0.0, 0.0, 0.0),
                 map_size=14.0, bce_sigma=0.1, delta=None, eikonal_weight=0.1, gs_sdf_weight=1e-3, visible_thr=0.1, mlp_mode=None,
                 eikonal_mode=None, align_weight=0.1, rgb_weight=0.8, dssim_weight=0.2, depth_weight=0.1, normal_weight=0.0,
                 isotropic_weight=0.0, delta_dev=None, bck_color=0, mask=None, depth_type=0, frame_sizes=None):
        """delta_dev: float32 CUDA tensor [1] read by every SDF call of [A] and [C] in place of the host scalar `delta` (the sample std the
        SDF stage adapts on the device, nsdf.SdfTrainer.std_dev); the ray-site forward then also evaluates the base variant into ray_y1.
        bck_color (k_bck_color: 0 black, 1 white, 2 random) and mask (bool / uint8 [H,W], [H,W,1] or [H,W,3] on the device, one for every
        frame): the render's background and the photometric loss's image mask (DESIGN 7o), in the joint step and in color_step. With
        bck_color 2 the render composites self.bg [1,H,W,3], which the caller fills before every render (gstrain.GsTrainer draws it).
        depth_type (k_depth_type): the depth of the normal-consistency term, 0 the expected depth, any other int the median depth.
        frame_sizes: the (W, H) of every frame the step will train or render (SplatRenderer; set_frame switches between them)."""
        check_photometric("GsSdfStep", bck_color, mask, H, W, device)
        self.median_depth = check_depth_type("GsSdfStep", depth_type)
        self.R = SplatRenderer(N, K, 1, W, H, device, isect_cap, sh_degree=sh_degree, frame_sizes=frame_sizes)
        self.bck_color, self.mask = int(bck_color), expand_mask(mask, H, W)
        self._bg_store = torch.zeros(3 * self.R.max_pixels, dtype=torch.float32, device=device) if self.bck_color == 2 else None
        self.bg = self._bg_store[:3 * H * W].view(1, H, W, 3) if self.bck_color == 2 else None
        self.dev, self.N, self.n_ray = device, N, n_ray_samples
        self.cfg = dict(sdf_net_cfg)
        self.origin, self.inv_size = tuple(origin), 1.0 / map_size
        self.bce_isigma, self.delta = 1.0 / bce_sigma, (delta if delta is not None else bce_sigma)  # k_sample_std = k_bce_sigma
        self.eik_w, self.gs_sdf_w, self.vis_thr = eikonal_weight, gs_sdf_weight, visible_thr
        # photometric loss: k_rgb_weight * L1 + k_dssim_weight * (1 - SSIM) (config/base.yaml:35-36) (+ an L1 on the expected depth)
        self.rgb_w, self.dssim_w, self.depth_w = rgb_weight, dssim_weight, depth_weight
        # k_render_normal_weight / k_isotropic_weight (config/base.yaml:43-46: 0.01 / 0.05; the normal term from iteration 3000 on)
        self.normal_w, self.iso_w = normal_weight, isotropic_weight
        self.valid_mask = None       # [cap] uint8 octree validity of the splat samples (LocalMap::get_valid_mask) or None
        self.octree = None
        self.keep_shadows = False    # True: the caller (GsSdfTrainer's Adam) keeps table_half / mlp_packed current and zeroes the gradients
        f32 = dict(dtype=torch.float32, device=device)
        probe = cabi.sdf_net(torch.zeros(1, **f32), torch.zeros(1, **f32), **self.cfg)
        self.n_table, self.n_mlp = cabi.sdf_table_params(probe), cabi.sdf_mlp_params(probe)
        self.table_half = torch.empty(self.n_table, dtype=torch.float16, device=device)
        # decoder arithmetic: tensor cores (wgmma, sdf_tc.cu) wherever the configuration allows it, else fp32 CUDA cores
        tc_ok = self.cfg.get("hidden_dim", 64) == 64 and self.cfg.get("n_hidden", 3) <= 3
        self.mlp_mode = (1 if tc_ok else 0) if mlp_mode is None else int(mlp_mode)
        self.mlp_packed = torch.empty(cabi.sdf_mlp_packed_bytes(probe), dtype=torch.uint8, device=device) if self.mlp_mode == 1 else None
        # eikonal: 1 = on the analytic gradient + align loss (reference default, config/base.yaml:13,32; fused tensor-core kernel only),
        # 0 = on the 6-offset numerical gradient (k_numerical_grad)
        self.eik_mode = (1 if self.mlp_mode == 1 else 0) if eikonal_mode is None else int(eikonal_mode)
        assert self.eik_mode == 0 or self.mlp_mode == 1, "the analytic eikonal path lives in the fused tensor-core kernel (mlp_mode 1)"
        self.align_w = float(align_weight) if self.eik_mode == 1 else 0.0
        if delta_dev is not None:
            if self.eik_mode != 1:
                raise ValueError("GsSdfStep: a device delta needs eikonal_mode 1 (the numerical-gradient path has no device-delta entry)")
            if not (isinstance(delta_dev, torch.Tensor) and delta_dev.is_cuda and delta_dev.dtype == torch.float32 and delta_dev.numel() == 1):
                raise ValueError("GsSdfStep: delta_dev must be a float32 CUDA tensor [1]")
        self.delta_dev = delta_dev
        # flat gradient: [splat | (pad to an even offset: the table gradient takes 8-byte vector REDs) | table | mlp]
        n_splat = self.R.flat_grad.numel()
        t0 = (n_splat + 1) // 2 * 2
        self.flat_grad = torch.zeros(t0 + self.n_table + self.n_mlp, **f32)
        self._rebind_splat_grads(n_splat)
        self.table_grad = self.flat_grad[t0:t0 + self.n_table]
        self.mlp_grad = self.flat_grad[t0 + self.n_table:]
        e = lambda *s: torch.empty(*s, **f32)
        self.ray_sdf, self.ray_y1, self.ray_vs, self.ray_vy = e(7 * n_ray_samples), e(7 * n_ray_samples), e(7 * n_ray_samples), e(7 * n_ray_samples)
        cap = self.R.cap
        self.gs_sdf, self.gs_y1, self.gs_vs, self.gs_vy = e(7 * cap), e(7 * cap), e(7 * cap), e(7 * cap)
        self.v_samples = e(cap, 3)
        self.sdf_loss = torch.zeros(1, **f32)
        self.n_gate = torch.zeros(1, dtype=torch.int32, device=device)
        # compact copies of the gated splat samples (the reference's index_select, neural_mapping.cpp:433-437)
        self.compact_gate = True
        self.gate_idx = torch.empty(cap, dtype=torch.int32, device=device)
        self.gate_x, self.gate_w, self.gate_vx = e(cap, 3), e(cap), e(cap, 3)
        self.gate_ws = cabi.Workspace(device)
        # overlap: the SDF-only work of a step (sample generation, [A], [C]) is enqueued on a second stream and runs concurrently with the
        # render: [A] beside projection .. raster forward, [C] (which needs the forward's visibilities) beside losses .. SH backward; the
        # projection backward waits for [C]'s dL/d sample. Same kernels, same results; only the schedule changes.
        self.overlap = False
        # with `overlap`: False keeps sample generation + [A] on the caller's stream (ahead of the render) and only [C] goes to the second
        # stream -- what a data-parallel caller wants while a dense gradient all-reduce of the previous step is still in flight, which
        # [A] then covers (parallel.DataParallelStep sets it per step)
        self.overlap_ray_stage = True
        self.sdf_stream_priority = 0
        self._side = None
        self._ev_fwd, self._ev_c = torch.cuda.Event(), torch.cuda.Event()

    def set_frame(self, W, H, mask=None):
        """Train / render W x H frames from here on (SplatRenderer.set_frame): the renderer's per-pixel buffers and the background
        (bck_color 2, drawn by the caller after this) become views of that size. mask: a new image mask of that size (check_photometric);
        without one, the current mask stays and must have that size."""
        if mask is not None:
            check_photometric("GsSdfStep.set_frame", self.bck_color, mask, int(H), int(W), self.dev)
        elif self.mask is not None and tuple(self.mask.shape[:2]) != (int(H), int(W)):
            raise ValueError(f"GsSdfStep.set_frame: the image mask is {tuple(self.mask.shape[:2])}, the frame {int(H)}x{int(W)} (H x W)")
        self.view_frame(W, H)
        if mask is not None:
            self.mask = expand_mask(mask, self.R.H, self.R.W)

    def view_frame(self, W, H):
        """set_frame without the mask: for renders outside the loss."""
        self.R.set_frame(W, H)
        if self._bg_store is not None:
            self.bg = self._bg_store[:3 * self.R.H * self.R.W].view(1, self.R.H, self.R.W, 3)

    @contextlib.contextmanager
    def sdf_stage(self):
        """Stream context for work that touches SDF-side state only (ray sample generation, stage [A]). Without `overlap` it is the
        caller's stream; with it, the second stream, ordered after everything the caller's stream has enqueued so far (the previous step's
        optimiser update included)."""
        if not (self.overlap and self.overlap_ray_stage):
            yield
            return
        side = self._side_stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            yield

    def _side_stream(self):
        if self._side is None:
            self._side = torch.cuda.Stream(device=self.dev, priority=self.sdf_stream_priority)
        return self._side

    # + 2 DSSIM kernels + table cast + decoder weight image + gate count + 2 x (7-variant forward, fused train) (mlp_mode 1) + the catch-up of
    # the visible SH rows that GsSdfTrainer's lazy Adam launches before the SH forward (SH degree > 0)
    KERNELS_PER_STEP = SplatRenderer.KERNELS_PER_STEP + 10

    def _rebind_splat_grads(self, n_splat):
        R, N, K = self.R, self.R.N, self.R.K
        R.flat_grad = self.flat_grad[:n_splat]
        o = [0, N * 3, N * 7, N * 10, N * 11, N * 11 + N * K * 3]
        fg = R.flat_grad
        R.v_means, R.v_quats, R.v_scales = fg[o[0]:o[1]].view(N, 3), fg[o[1]:o[2]].view(N, 4), fg[o[2]:o[3]].view(N, 3)
        R.v_opac, R.v_sh = fg[o[3]:o[4]], fg[o[4]:o[5]].view(N, K, 3)

    def refresh_table(self, table_f32):
        cabi.sdf_table_to_half(table_f32, self.table_half)

    def set_octree(self, octree):
        """OctreeAS of the occupancy map: stage [C] then also gates the splat samples by LocalMap::get_valid_mask (neural_mapping.cpp:432)."""
        self.octree = octree
        self.valid_mask = torch.zeros(self.R.cap, dtype=torch.uint8, device=self.dev) if octree is not None else None

    def _coupling_compact(self, net, samples, n_live, on_sdf_grads_ready):
        """[C] like the reference: select the gated samples first, evaluate the SDF network on them only, scatter dL/d sample back"""
        R, cap = self.R, self.R.cap
        cabi.sdf_gate_compact(cap, samples, self.gate_idx, self.gate_x, self.n_gate, self.gate_ws, visibilities=R.r["visibilities"],
                              visible_thr=self.vis_thr, valid_mask=self.valid_mask, weights=R.p["sample_weights"], w_out=self.gate_w,
                              n_live=n_live)
        if self.eik_mode == 1 and self.delta_dev is not None:
            if self.align_w > 0:
                cabi.sdf_fwd_dev(net, self.gate_x, self.gs_sdf, self.delta_dev, n_variants=7, n_live=self.n_gate, skip_base_variant=True)
            cabi.sdf_train_dev(net, self.gate_x, 1, self.delta_dev, None, self.gate_w, self.bce_isigma, 0.0, self.eik_w, self.gs_sdf_w,
                               self.sdf_loss, self.table_grad, self.mlp_grad, self.gate_vx, n_live=self.n_gate, eikonal_mode=1,
                               align_weight=self.align_w, sdf_variants=self.gs_sdf if self.align_w > 0 else None)
        elif self.eik_mode == 1:
            if self.align_w > 0:
                cabi.sdf_fwd(net, self.gate_x, self.gs_sdf, None, None, n_variants=7, delta=self.delta, n_live=self.n_gate,
                             skip_base_variant=True)
            cabi.sdf_train(net, self.gate_x, 1, self.delta, None, self.gate_w, self.bce_isigma, 0.0, self.eik_w, self.gs_sdf_w,
                           self.sdf_loss, self.table_grad, self.mlp_grad, self.gate_vx, n_live=self.n_gate, eikonal_mode=1,
                           align_weight=self.align_w, sdf_variants=self.gs_sdf if self.align_w > 0 else None)
        else:
            cabi.sdf_train(net, self.gate_x, 7, self.delta, None, self.gate_w, self.bce_isigma, 0.0, self.eik_w, self.gs_sdf_w,
                           self.sdf_loss, self.table_grad, self.mlp_grad, self.gate_vx, n_live=self.n_gate)
        cabi.scatter_rows3(cap, self.gate_idx, self.n_gate, self.gate_vx, self.v_samples, n_live=n_live)
        R._mark("sdf_splat_samples[C]")
        if on_sdf_grads_ready is not None:  # (NCCL orders itself after the stream that is current here)
            on_sdf_grads_ready(self.flat_grad[self.table_grad.storage_offset():])

    def step(self, scene, table_f32, mlp, viewmats, Ks, gt_image, ray_xyz, ray_gt_sdf, randns=None, on_sdf_grads_ready=None,
             before_render=None, ray_n_live=None):
        """ray_n_live: device int32 (e.g. RaySampler.counts): only the first *ray_n_live rows of ray_xyz / ray_gt_sdf are samples.
        ray_xyz None: no SDF stage [A] (detach_sdf_grad: the SDF is frozen)."""
        """Hooks for a data-parallel caller (both optional):
        on_sdf_grads_ready(table_and_mlp_grad): the hash-table / decoder gradients are final (after [C]) -> start reducing them while the
            render backward [D] is still running.
        before_render(): called after stage [A] and before anything touches the splat parameters or their gradient segment. Stage [A]
            depends on the SDF parameters only, so the PREVIOUS step's splat-gradient all-reduce (and splat optimiser step) may still be
            in flight while [A] runs; the caller waits for them here."""
        R, n_ray, cap = self.R, self.n_ray, self.R.cap
        R._mark("start")
        with self.sdf_stage():
            # fp32 master -> fp16 shadow once per step (the optimiser moved the master; the reference casts on EVERY forward)
            if not self.keep_shadows:
                cabi.sdf_table_to_half(table_f32, self.table_half)
                if self.mlp_mode == 1:  # bf16 hi/mid/lo weight image for the tensor-core decoder, also once per step
                    cabi.sdf_mlp_pack(cabi.sdf_net(self.table_half, mlp, **self.cfg), self.mlp_packed)
            net = cabi.sdf_net(self.table_half, mlp, origin=self.origin, inv_size=self.inv_size, mlp_mode=self.mlp_mode,
                               mlp_packed=self.mlp_packed, **self.cfg)
            t0 = self.table_grad.storage_offset()
            if not self.keep_shadows:
                self.flat_grad[t0:].zero_()  # table + decoder segment; the splat segment is cleared after before_render()
            self.sdf_loss.zero_()
            # [A] SDF stage on the ray samples (tensor-core mode: forward + losses + backward fused in one kernel)
            if ray_xyz is None:
                pass
            elif self.delta_dev is not None:  # base variant included: y1 of the base rows feeds the sample-std update (gssdf_sdf_adapt)
                cabi.sdf_fwd_dev(net, ray_xyz, self.ray_sdf, self.delta_dev, y1=self.ray_y1, n_variants=7 if self.align_w > 0 else 1,
                                 n_live=ray_n_live)
                cabi.sdf_train_dev(net, ray_xyz, 1, self.delta_dev, ray_gt_sdf, None, self.bce_isigma, 1.0, self.eik_w, 0.0, self.sdf_loss,
                                   self.table_grad, self.mlp_grad, None, eikonal_mode=1, align_weight=self.align_w,
                                   sdf_variants=self.ray_sdf if self.align_w > 0 else None, n_live=ray_n_live)
            elif self.mlp_mode == 1:
                if self.eik_mode == 1:  # reference default: forward-only pass over the 7 variants (numerical gradient of the align loss),
                                        # then forward + losses + backward + double backward on the base points only
                    if self.align_w > 0:
                        cabi.sdf_fwd(net, ray_xyz, self.ray_sdf, None, None, n_variants=7, delta=self.delta, skip_base_variant=True, n_live=ray_n_live)
                    cabi.sdf_train(net, ray_xyz, 1, self.delta, ray_gt_sdf, None, self.bce_isigma, 1.0, self.eik_w, 0.0, self.sdf_loss,
                                   self.table_grad, self.mlp_grad, None, eikonal_mode=1, align_weight=self.align_w,
                                   sdf_variants=self.ray_sdf if self.align_w > 0 else None, n_live=ray_n_live)
                else:
                    cabi.sdf_train(net, ray_xyz, 7, self.delta, ray_gt_sdf, None, self.bce_isigma, 1.0, self.eik_w, 0.0, self.sdf_loss,
                                   self.table_grad, self.mlp_grad, None, n_live=ray_n_live)
            else:
                cabi.sdf_fwd(net, ray_xyz, self.ray_sdf, self.ray_y1, None, n_variants=7, delta=self.delta, n_live=ray_n_live)
                cabi.sdf_loss(n_ray, 7, self.ray_sdf, self.ray_y1, ray_gt_sdf, None, self.bce_isigma, 1.0, self.eik_w, 0.0, self.delta, self.sdf_loss,
                              self.ray_vs, self.ray_vy, n_live=ray_n_live)
                cabi.sdf_bwd(net, ray_xyz, self.ray_vs, self.ray_vy, self.table_grad, self.mlp_grad, None, n_variants=7, delta=self.delta,
                             n_live=ray_n_live)
            R._mark("sdf_ray_samples[A]")
        if before_render is not None:
            before_render()
        if not self.keep_shadows:
            self.flat_grad[:t0].zero_()
        # [B] render
        R.forward(scene["means"], scene["quats"], scene["scales"], scene["opacities"], scene["sh"], viewmats, Ks, randns,
                  raw=scene.get("raw"), bck_color=self.bck_color, bg=self.bg)
        # [C] coupling on the stochastic splat samples (rows < nnz, counted on the device)
        samples, n_live = R.p["samples"], R.counts  # counts[0] == nnz
        # the reference's sample gate: vis > visible_thr (& octree validity), counted on the device (no nonzero() / .item() sync)
        side = self._side_stream() if self.overlap else None
        assert side is None or (self.compact_gate and self.mlp_mode == 1), "overlap needs the compact-gate tensor-core path"
        if side is not None:  # [C] needs the forward's visibilities / samples: the second stream picks up after the raster forward
            self._ev_fwd.record()
            side.wait_event(self._ev_fwd)
        with (torch.cuda.stream(side) if side is not None else contextlib.nullcontext()):
            if getattr(self, "octree", None) is not None:
                self.octree.valid_mask(samples, self.valid_mask, n_live=n_live)
            if self.compact_gate and self.mlp_mode == 1:
                self._coupling_compact(net, samples, n_live, None)
                if side is not None:
                    self._ev_c.record(side)  # dL/d sample is ready: all the projection backward waits for
                if on_sdf_grads_ready is not None:  # the hash-table / decoder gradients are final (NCCL, or the caller's SDF optimiser
                    on_sdf_grads_ready(self.flat_grad[self.table_grad.storage_offset():])  # step, order themselves after the stream current here)
        if self.compact_gate and self.mlp_mode == 1:
            wait_c = (lambda: torch.cuda.current_stream().wait_event(self._ev_c)) if side is not None else None
            loss = R.backward(scene["means"], scene["quats"], scene["scales"], scene["opacities"], scene["sh"], viewmats, Ks, gt_image, randns,
                              v_samples=self.v_samples, zero_grads=False, raw=scene.get("raw"), w_rgb=self.rgb_w, w_depth=self.depth_w,
                              w_dssim=self.dssim_w, w_normal=self.normal_w, w_isotropic=self.iso_w, before_projection_bwd=wait_c,
                              bck_color=self.bck_color, bg=self.bg, mask=self.mask, median_depth=self.median_depth)
            return loss, self.sdf_loss
        cabi.sdf_gate_count(cap, self.n_gate, visibilities=R.r["visibilities"], visible_thr=self.vis_thr, valid_mask=self.valid_mask,
                            n_live=n_live)
        gate = dict(valid_mask=self.valid_mask, n_gate=self.n_gate)
        if self.mlp_mode == 1 and self.delta_dev is not None:
            if self.align_w > 0:
                cabi.sdf_fwd_dev(net, samples, self.gs_sdf, self.delta_dev, n_variants=7, n_live=n_live, skip_base_variant=True)
            cabi.sdf_train_dev(net, samples, 1, self.delta_dev, None, R.p["sample_weights"], self.bce_isigma, 0.0, self.eik_w, self.gs_sdf_w,
                               self.sdf_loss, self.table_grad, self.mlp_grad, self.v_samples, visibilities=R.r["visibilities"],
                               visible_thr=self.vis_thr, n_live=n_live, eikonal_mode=1, align_weight=self.align_w,
                               sdf_variants=self.gs_sdf if self.align_w > 0 else None, **gate)
        elif self.mlp_mode == 1:
            if self.eik_mode == 1:
                if self.align_w > 0:
                    cabi.sdf_fwd(net, samples, self.gs_sdf, None, None, n_variants=7, delta=self.delta, n_live=n_live, skip_base_variant=True)
                cabi.sdf_train(net, samples, 1, self.delta, None, R.p["sample_weights"], self.bce_isigma, 0.0, self.eik_w, self.gs_sdf_w,
                               self.sdf_loss, self.table_grad, self.mlp_grad, self.v_samples, visibilities=R.r["visibilities"],
                               visible_thr=self.vis_thr, n_live=n_live, eikonal_mode=1, align_weight=self.align_w,
                               sdf_variants=self.gs_sdf if self.align_w > 0 else None, **gate)
            else:
                cabi.sdf_train(net, samples, 7, self.delta, None, R.p["sample_weights"], self.bce_isigma, 0.0, self.eik_w, self.gs_sdf_w,
                               self.sdf_loss, self.table_grad, self.mlp_grad, self.v_samples, visibilities=R.r["visibilities"],
                               visible_thr=self.vis_thr, n_live=n_live, **gate)
        else:
            cabi.sdf_fwd(net, samples, self.gs_sdf, self.gs_y1, None, n_variants=7, delta=self.delta, n_live=n_live)
            cabi.sdf_loss(cap, 7, self.gs_sdf, self.gs_y1, None, R.p["sample_weights"], self.bce_isigma, 0.0, self.eik_w, self.gs_sdf_w, self.delta,
                          self.sdf_loss, self.gs_vs, self.gs_vy, visibilities=R.r["visibilities"], visible_thr=self.vis_thr, n_live=n_live,
                          **gate)
            cabi.sdf_bwd(net, samples, self.gs_vs, self.gs_vy, self.table_grad, self.mlp_grad, self.v_samples, n_variants=7, delta=self.delta,
                         n_live=n_live)
        R._mark("sdf_splat_samples[C]")
        if on_sdf_grads_ready is not None:
            on_sdf_grads_ready(self.flat_grad[self.table_grad.storage_offset():])
        # [D] photometric loss + backward of the render, with the coupling gradient entering through the samples
        loss = R.backward(scene["means"], scene["quats"], scene["scales"], scene["opacities"], scene["sh"], viewmats, Ks, gt_image, randns,
                          v_samples=self.v_samples, zero_grads=False, raw=scene.get("raw"), w_rgb=self.rgb_w, w_depth=self.depth_w,
                          w_dssim=self.dssim_w, w_normal=self.normal_w, w_isotropic=self.iso_w, bck_color=self.bck_color, bg=self.bg,
                          mask=self.mask, median_depth=self.median_depth)
        return loss, self.sdf_loss


def sh_sweep_step(t):
    """Adam steps at which the lazy SH row groups update every row instead of the visible ones: one per window, so that no row is ever
    more than ADAM_WINDOW - 1 steps behind and every replayed step's scalars are still in the window."""
    return t % cabi.ADAM_WINDOW == 0


class GsSdfTrainer(GsSdfStep):
    """GsSdfStep + the optimiser step of the reference loop (`zero_grad; backward; Adam.step()`, neural_mapping.cpp:466-469): owns ONE
    flat fp32 parameter buffer with exactly the layout of the flat gradient

        [ offsets N*3 | quaternion N*4 | scaling N*3 | opacity N | features_dc N*3 | features_rest N*(K-1)*3 | pad | hash table | decoder ]

    plus Adam's two moment buffers, and runs `gssdf_adam_step` over its parameter groups (learning rates of
    neural_gaussian.cpp:434-449 and config/base.yaml:25; eps 1e-15). The same kernel zeroes the gradient, refreshes the fp16 shadow of
    the hash table and re-packs the decoder's bf16 operand image, so a training step launches no cast / pack / memset kernels.
    `anchors` are not optimised (register_parameter(..., false), neural_gaussian.cpp:426).

    Lazy SH rows (SH degree > 0, single process): features_dc / features_rest are Adam ROW groups. A step's camera gives an SH gradient
    to its visible rows only, so adam_all updates just those rows, a catch-up launch before the SH forward brings the rows it reads up
    to date (the step's one launch more, counted in GsSdfStep.KERNELS_PER_STEP), and every
    ADAM_WINDOW steps one sweep updates every row (DESIGN.md section 7c). Results are bit-identical to the dense update. `params`,
    `exp_avg` and `exp_avg_sq` bring every row current before they are returned; code inside the step uses `_params` & co. and the
    `scene` views, which may hold stale SH rows."""

    def __init__(self, *a, spatial_scale=1.0, sdf_lr=5e-3, n_live=None, **kw):
        """The first positional argument N is the row CAPACITY of the splat buffers; n_live (default N) splats are in use. Densification
        (gssdf_b200/densify.py) changes n_live between steps; every segment of the flat buffers keeps its capacity-based offset."""
        super().__init__(*a, **kw)
        N, K = self.R.N, self.R.K
        f32 = dict(dtype=torch.float32, device=self.dev)
        n = self.flat_grad.numel()
        self._params, self._exp_avg, self._exp_avg_sq = torch.zeros(n, **f32), torch.zeros(n, **f32), torch.zeros(n, **f32)
        self.lazy_sh = K > 1
        self.sh_last = torch.zeros(N, dtype=torch.int32, device=self.dev)  # Adam step at which each SH row was last brought current
        self.sh_replay = cabi.AdamReplay(self.sh_last)
        self._sh_stale = False  # True: some SH rows may be behind t_splat
        self.t0 = self.table_grad.storage_offset()
        self.seg_off = [0, N * 3, N * 7, N * 10, N * 11, N * 14, N * 11 + N * K * 3]  # offsets|quaternion|scaling|opacity|dc|rest
        self.seg_w = [3, 4, 3, 1, 3, 3 * (K - 1)]
        self.lr = [1.6e-4 * spatial_scale, 0.001, 0.005, 0.05, 0.0025, 0.0025 / 20.0]  # neural_gaussian.cpp:434-449
        self.sdf_lr = sdf_lr
        self.anchors_buf = torch.zeros(N, 3, **f32)
        self.keep_shadows = True
        self.t_splat = self.t_sdf = 0
        self.t_sh = 0  # the SH groups' Adam step: t_splat unless colour initialisation stepped them alone (adam_sh)
        self._net = None
        self.l2_persist = False  # off by default: the 30.5 MB table fits the 50 MB L2 without a persistence window
        self.N_cap = N
        self.N_live = None
        self.set_live(N if n_live is None else n_live)

    # the three flat buffers: reading one from outside the step brings every SH row current first
    @property
    def params(self):
        self.flush_sh()
        return self._params

    @params.setter
    def params(self, t):
        self._params = t

    @property
    def exp_avg(self):
        self.flush_sh()
        return self._exp_avg

    @exp_avg.setter
    def exp_avg(self, t):
        self._exp_avg = t

    @property
    def exp_avg_sq(self):
        self.flush_sh()
        return self._exp_avg_sq

    @exp_avg_sq.setter
    def exp_avg_sq(self, t):
        self._exp_avg_sq = t

    def flush_sh(self):
        """Replay the skipped zero-gradient Adam steps of every stale SH row up to t_sh (one launch; nothing when all are current)."""
        if not self._sh_stale:
            return
        self._sh_stale = False
        cabi.adam_step(self._params, self.flat_grad, self._exp_avg, self._exp_avg_sq, self._sh_groups(), self.t_sh,
                       replay=self.sh_replay, replay_only=True)

    def _sh_groups(self):
        o, w, n = self.seg_off, self.seg_w, self.N_live
        return [(o[4], n * w[4], self.lr[4], False, w[4]), (o[5], n * w[5], self.lr[5], False, w[5])]

    def _sh_catch_up(self):
        """Before the SH forward reads them: the rows of this step's camera get the zero-gradient steps they missed (one launch)."""
        if self.t_sh > 0:
            cabi.adam_step(self._params, self.flat_grad, self._exp_avg, self._exp_avg_sq, self._sh_groups(), self.t_sh,
                           replay=self.sh_replay, row_ids=self.R.p["gaussian_ids"], row_count=self.R.counts, row_cap=self.R.cap,
                           replay_only=True)

    def stamp_sh_current(self):
        """Every SH row holds its values at step t_sh (after load / a row remap of current rows)."""
        self.sh_last.fill_(self.t_sh)
        self._sh_stale = False

    def set_live(self, n_live):
        """(Re)bind the parameter views and Adam groups to the first n_live rows of every segment."""
        assert 0 <= n_live <= self.N_cap
        if self.N_live is not None and int(n_live) != self.N_live:  # rows enter or leave the row groups: all rows current first
            self.flush_sh()
            self.stamp_sh_current()
        self.N_live = n = int(n_live)
        o, w, pv, K = self.seg_off, self.seg_w, self._params, self.R.K
        v = lambda s_, *shape: pv[o[s_]:o[s_] + n * w[s_]].view(n, *shape)
        self.anchors = self.anchors_buf[:n]
        catch_up = self._sh_catch_up if self.lazy_sh else None
        self.scene = dict(means=self.anchors, quats=v(1, 4), scales=v(2, 3), opacities=pv[o[3]:o[3] + n], sh=v(4, 1, 3),
                          raw=dict(offsets=v(0, 3), sh_rest=v(5, K - 1, 3) if K > 1 else None, sh_catch_up=catch_up))
        # (offset, count, lr, half_shadow, row_width): features_dc / features_rest are row groups on the lazy path
        self.splat_groups = [(o[i], n * w[i], self.lr[i], False, w[i] if (self.lazy_sh and i >= 4) else 0)
                             for i in range(6) if w[i] > 0 and n > 0]
        self.splat_group_is_sh = [i >= 4 for i in range(6) if w[i] > 0 and n > 0]
        t0 = self.t0
        self.sdf_groups = [(t0, self.n_table, self.sdf_lr, True), (t0 + self.n_table, self.n_mlp, self.sdf_lr, False)]
        self.table, self.mlp = pv[t0:t0 + self.n_table], pv[t0 + self.n_table:]
        if self._net is not None:
            self._net = cabi.sdf_net(self.table_half, self.mlp, **self.cfg)

    def load(self, anchors, offsets, quats, log_scales, logit_opacities, features_dc, features_rest, table, mlp, sdf_exp_avg=None,
             sdf_exp_avg_sq=None, sdf_step=0):
        """sdf_exp_avg / sdf_exp_avg_sq ([table | decoder], e.g. nsdf.SdfTrainer's) and sdf_step: the SDF groups continue with those Adam
        moments and that step count (one optimiser spans both stages in the reference); without them the SDF moments start at zero."""
        if (sdf_exp_avg is None) != (sdf_exp_avg_sq is None) or (sdf_exp_avg is None and sdf_step != 0) or sdf_step < 0:
            raise ValueError("GsSdfTrainer.load: give both SDF moments with their step count, or neither")
        self.set_live(anchors.shape[0])
        sc = self.scene
        self.anchors.copy_(anchors)
        sc["raw"]["offsets"].copy_(offsets); sc["quats"].copy_(quats); sc["scales"].copy_(log_scales); sc["opacities"].copy_(logit_opacities)
        sc["sh"].copy_(features_dc.view_as(sc["sh"]))
        if sc["raw"]["sh_rest"] is not None:
            sc["raw"]["sh_rest"].copy_(features_rest)
        self.table.copy_(table); self.mlp.copy_(mlp)
        self._exp_avg.zero_(); self._exp_avg_sq.zero_(); self.flat_grad.zero_()
        self.t_splat = self.t_sdf = self.t_sh = 0
        if sdf_exp_avg is not None:
            n_sdf = self.n_table + self.n_mlp
            self._exp_avg[self.t0:self.t0 + n_sdf].copy_(sdf_exp_avg.reshape(-1))
            self._exp_avg_sq[self.t0:self.t0 + n_sdf].copy_(sdf_exp_avg_sq.reshape(-1))
            self.t_sdf = int(sdf_step)
        self.stamp_sh_current()
        cabi.sdf_table_to_half(self.table, self.table_half)
        self._net = cabi.sdf_net(self.table_half, self.mlp, **self.cfg)
        if self.mlp_mode == 1:
            cabi.sdf_mlp_pack(self._net, self.mlp_packed)
        if self.l2_persist:  # the 30.5 MB fp16 table stays in L2 across the optimiser's streaming pass (SURVEY 7.6)
            cabi.l2_persist(self.table_half)

    def _adam_call(self, groups, t, grad_scale, sdf, rows=False):
        """rows: the SH row groups visit the rows of this step's camera only (else every row, a sweep)"""
        row = dict(row_ids=self.R.p["gaussian_ids"], row_count=self.R.counts, row_cap=self.R.cap) if rows else {}
        cabi.adam_step(self._params, self.flat_grad, self._exp_avg, self._exp_avg_sq, groups, t, grad_scale=grad_scale, zero_grads=True,
                       table_half=self.table_half if sdf else None, net=self._net if (sdf and self.mlp_mode == 1) else None,
                       mlp_packed=self.mlp_packed if (sdf and self.mlp_mode == 1) else None, replay=self.sh_replay, **row)
        self._sh_stale = rows

    def _next_splat_step(self):
        self.t_splat += 1
        self.t_sh += 1
        self.sh_replay.push(self.t_sh, self.lr[4], self.lr[5])
        return self.t_splat

    def adam_sdf(self, grad_scale=1.0):
        self.t_sdf += 1
        self._adam_call(self.sdf_groups, self.t_sdf, grad_scale, True)
        self.R._mark("adam_sdf")

    def adam_splat(self, grad_scale=1.0):
        """Data parallel: after an exchange every rank may hold gradients on any row, so the SH row groups sweep every row."""
        t = self._next_splat_step()
        self._adam_call(self.splat_groups, t, grad_scale, False)
        self.R._mark("adam_splat")

    def adam_all(self, grad_scale=1.0):
        """Single-GPU: one launch over all seven groups (+ the decoder re-pack). The SH row groups visit the rows the step's camera
        saw (the only rows with an SH gradient) and sweep every row once per ADAM_WINDOW steps, so that no row falls a window behind."""
        self.t_sdf += 1
        t = self._next_splat_step()
        assert self.t_sdf == t == self.t_sh
        self._adam_call(self.splat_groups + self.sdf_groups, t, grad_scale, True, rows=self.lazy_sh and not sh_sweep_step(t))
        self.R._mark("adam")

    def train_step(self, viewmats, Ks, gt_image, ray_xyz, ray_gt_sdf, randns=None, on_sdf_grads_ready=None, before_render=None,
                   ray_n_live=None):
        return self.step(self.scene, self.table, self.mlp, viewmats, Ks, gt_image, ray_xyz, ray_gt_sdf, randns,
                         on_sdf_grads_ready=on_sdf_grads_ready, before_render=before_render, ray_n_live=ray_n_live)

    # ---- per-group clocks (gstrain.GsTrainer: the SDF groups arrive with the SDF stage's steps, the SH groups with colour
    # initialisation's) -------------------------------------------------------------------------------------------------------------
    def adam_clocks(self, sdf=True):
        """adam_all with every group at its own step count: SDF groups t_sdf + 1, SH groups t_sh + 1, the other splat groups t_splat + 1
        (gssdf_adam_step_clocks, one launch). sdf=False leaves the SDF groups out (detach_sdf_grad)."""
        t = self._next_splat_step()
        steps = [self.t_sh if is_sh else t for is_sh in self.splat_group_is_sh]
        groups = list(self.splat_groups)
        if sdf:
            self.t_sdf += 1
            groups += self.sdf_groups
            steps += [self.t_sdf] * len(self.sdf_groups)
        self._adam_clocks_call(groups, steps, sdf, rows=self.lazy_sh and not sh_sweep_step(self.t_sh))
        self.R._mark("adam")

    def adam_sh(self):
        """Adam over the SH groups alone at the next SH step (colour initialisation: the structure and the SDF are frozen)."""
        self.t_sh += 1
        self.sh_replay.push(self.t_sh, self.lr[4], self.lr[5])
        groups = [g for g, is_sh in zip(self.splat_groups, self.splat_group_is_sh) if is_sh]
        self._adam_clocks_call(groups, [self.t_sh] * len(groups), False, rows=self.lazy_sh and not sh_sweep_step(self.t_sh))

    def _adam_clocks_call(self, groups, steps, sdf, rows):
        row = dict(row_ids=self.R.p["gaussian_ids"], row_count=self.R.counts, row_cap=self.R.cap) if rows else {}
        cabi.adam_step_clocks(self._params, self.flat_grad, self._exp_avg, self._exp_avg_sq, groups, steps, zero_grads=True,
                              table_half=self.table_half if sdf else None, net=self._net if (sdf and self.mlp_mode == 1) else None,
                              mlp_packed=self.mlp_packed if (sdf and self.mlp_mode == 1) else None, replay=self.sh_replay, **row)
        self._sh_stale = rows

    def color_step(self, viewmats, Ks, gt_image):
        """One colour-initialisation iteration (gs_train_batch_iter(i, false) + Adam, neural_mapping.cpp:377-382): render at the current
        SH degree, the photometric loss alone (L1 + DSSIM: no SDF stage, no coupling, no normal, depth or isotropic term), the backward
        down to the SH coefficients (the frozen structure's projection backward is skipped) and Adam over the SH groups. The structure's
        gradient segments are left for the caller to clear."""
        R, sc = self.R, self.scene
        R.forward(sc["means"], sc["quats"], sc["scales"], sc["opacities"], sc["sh"], viewmats, Ks, raw=sc["raw"], bck_color=self.bck_color,
                  bg=self.bg)
        loss = R.backward(sc["means"], sc["quats"], sc["scales"], sc["opacities"], sc["sh"], viewmats, Ks, gt_image, zero_grads=False,
                          raw=sc["raw"], w_rgb=self.rgb_w, w_depth=0.0, w_dssim=self.dssim_w, projection_bwd=False, bck_color=self.bck_color,
                          bg=self.bg, mask=self.mask)
        self.adam_sh()
        return loss

    def sdf_net(self):
        """The gssdf_sdf_net of the current SDF (fp16 table shadow and decoder image as the optimiser keeps them), for operators run
        between steps (outlier removal)."""
        return cabi.sdf_net(self.table_half, self.mlp, origin=self.origin, inv_size=self.inv_size, mlp_mode=self.mlp_mode,
                            mlp_packed=self.mlp_packed, **self.cfg)
