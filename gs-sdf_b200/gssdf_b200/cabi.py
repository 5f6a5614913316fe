"""Thin functional layer: torch tensors (device memory + streams only) -> C ABI calls.

One function per entry point of include/gssdf_b200.h. Nothing here computes: every function fills an
args struct with raw device pointers and calls libgssdf_b200.so on torch's current CUDA stream.
"""
import math

import torch

from . import _lib
from ._lib import check, lib, make_args

COUNTS_INTS = 8  # sizeof(gssdf_counts) / 4
NNZ, N_ISECTS, NNZ_OVERFLOW, ISECT_OVERFLOW, MAX_TILE = 0, 1, 2, 3, 4


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _req(t, dtype, name):
    if t is None:
        return None
    if not t.is_cuda:
        raise ValueError(f"gssdf_b200: {name} must be a CUDA tensor")  # CHECK_CUDA (GSF/include/Common.h:12)
    if not t.is_contiguous():
        raise ValueError(f"gssdf_b200: {name} must be contiguous")  # CHECK_CONTIGUOUS (:13)
    if t.dtype != dtype:
        raise ValueError(f"gssdf_b200: {name} must be {dtype}, got {t.dtype}")
    return t


def new_counts(device, nnz=0, n_isects=0):
    c = torch.zeros(COUNTS_INTS, dtype=torch.int32, device=device)
    if nnz or n_isects:
        c[:2] = torch.tensor([nnz, n_isects], dtype=torch.int32)
    return c


class Workspace:
    """Grow-only device scratch buffer (the library itself never allocates)."""

    def __init__(self, device):
        self.device = device
        self.buf = None

    def get(self, nbytes):
        nbytes = max(int(nbytes), 256)
        if self.buf is None or self.buf.numel() < nbytes:
            self.buf = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        return self.buf


def project2dgs_fwd(means, quats, scales, viewmats, Ks, W, H, near, far, radius_clip, randns, cap, out, counts, ws,
                    opacities=None, mean_offsets=None, raw_params=False):
    """out: dict of capacity-sized tensors (camera_ids, gaussian_ids, radii, means2d, depths, ray_transforms,
    normals, samples, sample_weights, indptr)."""
    N, Cn = means.shape[0], viewmats.shape[0]
    f32 = torch.float32
    for n_, t in (("means", means), ("quats", quats), ("scales", scales), ("viewmats", viewmats), ("Ks", Ks)):
        _req(t, f32, n_)
    need = lib().gssdf_project2dgs_workspace_bytes(N, Cn)
    w = ws.get(need)
    a = make_args("gssdf_project2dgs_fwd_args", N=N, C=Cn, means=means, quats=quats, scales=scales, viewmats=viewmats,
                  Ks=Ks, image_width=W, image_height=H, near_plane=near, far_plane=far, radius_clip=radius_clip,
                  randns=_req(randns, f32, "randns"), opacities=_req(opacities, f32, "opacities"),
                  pt_opacities=out.get("pt_opacities") if opacities is not None else None, cap=cap,
                  camera_ids=out["camera_ids"],
                  gaussian_ids=out["gaussian_ids"], radii=out["radii"], means2d=out["means2d"], depths=out["depths"],
                  ray_transforms=out["ray_transforms"], normals=out["normals"], samples=out.get("samples"),
                  sample_weights=out.get("sample_weights"), indptr=out.get("indptr"), counts=counts, workspace=w,
                  workspace_bytes=w.numel(), mean_offsets=_req(mean_offsets, f32, "mean_offsets"), raw_params=int(bool(raw_params)))
    check(lib().gssdf_project2dgs_fwd(_lib.C.byref(a), _stream()))


def project2dgs_bwd(means, quats, scales, viewmats, Ks, W, H, cap, counts, camera_ids, gaussian_ids, ray_transforms,
                    randns, v_means2d, v_depths, v_ray_transforms, v_normals, v_samples, v_means, v_quats, v_scales,
                    v_pt_opacities=None, v_opacities=None, mean_offsets=None, raw_params=False, pt_opacities=None):
    a = make_args("gssdf_project2dgs_bwd_args", N=means.shape[0], C=viewmats.shape[0], means=means, quats=quats,
                  scales=scales, viewmats=viewmats, Ks=Ks, image_width=W, image_height=H, cap=cap, counts=counts,
                  camera_ids=camera_ids, gaussian_ids=gaussian_ids, ray_transforms=ray_transforms, randns=randns,
                  v_means2d=v_means2d, v_depths=v_depths, v_ray_transforms=v_ray_transforms, v_normals=v_normals,
                  v_samples=v_samples, v_means=v_means, v_quats=v_quats, v_scales=v_scales,
                  v_pt_opacities=v_pt_opacities, v_opacities=v_opacities, mean_offsets=mean_offsets, raw_params=int(bool(raw_params)),
                  pt_opacities=pt_opacities)
    check(lib().gssdf_project2dgs_bwd(_lib.C.byref(a), _stream()))


def view_colors_fwd(viewmats, means, sh, sh_degree, cap, counts, camera_ids, gaussian_ids, radii, colors, mean_offsets=None,
                    sh_rest=None):
    """sh_rest given: `sh` is features_dc [N,1,3], sh_rest features_rest [N,K-1,3] (no concatenated copy)."""
    K = sh.shape[1] + (sh_rest.shape[1] if sh_rest is not None else 0)
    a = make_args("gssdf_view_colors_fwd_args", N=means.shape[0], C=viewmats.shape[0], K=K,
                  sh_degree=sh_degree, viewmats=viewmats, means=means, sh=sh, cap=cap, counts=counts,
                  camera_ids=camera_ids, gaussian_ids=gaussian_ids, radii=radii, colors=colors, mean_offsets=mean_offsets,
                  sh_rest=sh_rest)
    check(lib().gssdf_view_colors_fwd(_lib.C.byref(a), _stream()))


def view_colors_bwd(viewmats, means, sh, sh_degree, cap, counts, camera_ids, gaussian_ids, radii, colors, v_colors,
                    v_sh, v_means, mean_offsets=None, sh_rest=None, v_sh_rest=None):
    K = sh.shape[1] + (sh_rest.shape[1] if sh_rest is not None else 0)
    a = make_args("gssdf_view_colors_bwd_args", N=means.shape[0], C=viewmats.shape[0], K=K,
                  sh_degree=sh_degree, viewmats=viewmats, means=means, sh=sh, cap=cap, counts=counts,
                  camera_ids=camera_ids, gaussian_ids=gaussian_ids, radii=radii, colors=colors, v_colors=v_colors,
                  v_sh=v_sh, v_means=v_means, mean_offsets=mean_offsets, sh_rest=sh_rest, v_sh_rest=v_sh_rest)
    check(lib().gssdf_view_colors_bwd(_lib.C.byref(a), _stream()))


def tile_encode(Cn, W, H, tile_size, cap, counts, means2d, radii, depths, camera_ids, isect_cap, tiles_per_gauss,
                isect_ids, flatten_ids, offsets, ws, conics=None):
    """conics=None: reference-identical lists. conics=[cap,8] (splat_conics): pairs whose exact footprint misses the tile are dropped
    before the sort (fused step; renders unchanged)."""
    need = lib().gssdf_tile_encode_workspace_bytes(Cn, W, H, tile_size, isect_cap)
    w = ws.get(need)
    a = make_args("gssdf_tile_encode_args", C=Cn, image_width=W, image_height=H, tile_size=tile_size, cap=cap,
                  counts=counts, means2d=means2d, radii=radii, depths=depths, camera_ids=camera_ids, isect_cap=isect_cap,
                  tiles_per_gauss=tiles_per_gauss, isect_ids=isect_ids, flatten_ids=flatten_ids, offsets=offsets,
                  workspace=w, workspace_bytes=w.numel(), conics=conics)
    check(lib().gssdf_tile_encode(_lib.C.byref(a), _stream()))


def splat_conics(cap, W, H, counts, ray_transforms, opacities, conics):
    a = make_args("gssdf_splat_conics_args", cap=cap, image_width=W, image_height=H, counts=counts, ray_transforms=ray_transforms,
                  opacities=opacities, conics=conics)
    check(lib().gssdf_splat_conics(_lib.C.byref(a), _stream()))


def raster2dgs_fwd(Cn, W, H, tile_size, channels, cap, counts, means2d, ray_transforms, colors, opacities, normals,
                   backgrounds, offsets, flatten_ids, out, ws, prof=None, isect_cap=None):
    isect_cap = int(flatten_ids.shape[0]) if isect_cap is None else int(isect_cap)
    need = lib().gssdf_raster2dgs_workspace_bytes(Cn, W, H, cap, _lib.C.c_int64(isect_cap))
    w = ws.get(need)
    a = make_args("gssdf_raster2dgs_fwd_args", C=Cn, image_width=W, image_height=H, tile_size=tile_size,
                  channels=channels, cap=cap, counts=counts, means2d=means2d, ray_transforms=ray_transforms,
                  colors=colors, opacities=opacities, normals=normals, backgrounds=backgrounds, offsets=offsets,
                  flatten_ids=flatten_ids, isect_cap=isect_cap, render_colors=out["render_colors"], render_depths=out["render_depths"],
                  render_alphas=out["render_alphas"], render_normals=out["render_normals"],
                  render_distort=out.get("render_distort"), render_median=out["render_median"], render_Ts=out.get("render_Ts"),
                  last_ids=out["last_ids"], median_ids=out["median_ids"], visibilities=out["visibilities"], workspace=w,
                  workspace_bytes=w.numel(), prof_start=prof[0].cuda_event if prof else None,
                  prof_stop=prof[1].cuda_event if prof else None)
    check(lib().gssdf_raster2dgs_fwd(_lib.C.byref(a), _stream()))


def raster2dgs_bwd(Cn, W, H, tile_size, channels, cap, counts, means2d, ray_transforms, colors, opacities, normals,
                   backgrounds, offsets, flatten_ids, render_alphas, render_Ts, last_ids, median_ids, v_render_colors,
                   v_render_depths, v_render_alphas, v_render_normals, v_render_median, out, ws, v_render_distort=None,
                   prof=None, isect_cap=None, reuse_fwd=False):
    isect_cap = int(flatten_ids.shape[0]) if isect_cap is None else int(isect_cap)
    need = lib().gssdf_raster2dgs_bwd_workspace_bytes(Cn, W, H, cap, _lib.C.c_int64(isect_cap))
    w = ws.get(need)
    a = make_args("gssdf_raster2dgs_bwd_args", C=Cn, image_width=W, image_height=H, tile_size=tile_size,
                  channels=channels, cap=cap, counts=counts, means2d=means2d, ray_transforms=ray_transforms,
                  colors=colors, opacities=opacities, normals=normals, backgrounds=backgrounds, offsets=offsets,
                  flatten_ids=flatten_ids, isect_cap=isect_cap, reuse_fwd=int(bool(reuse_fwd)), render_alphas=render_alphas,
                  render_Ts=render_Ts, last_ids=last_ids,
                  median_ids=median_ids, v_render_colors=v_render_colors, v_render_depths=v_render_depths,
                  v_render_alphas=v_render_alphas, v_render_normals=v_render_normals, v_render_distort=v_render_distort,
                  v_render_median=v_render_median, v_means2d=out.get("v_means2d"), v_means2d_abs=out.get("v_means2d_abs"),
                  v_ray_transforms=out["v_ray_transforms"], v_colors=out["v_colors"], v_opacities=out["v_opacities"],
                  v_normals=out["v_normals"], v_densify=out.get("v_densify"), workspace=w, workspace_bytes=w.numel(),
                  prof_start=prof[0].cuda_event if prof else None, prof_stop=prof[1].cuda_event if prof else None)
    check(lib().gssdf_raster2dgs_bwd(_lib.C.byref(a), _stream()))


def render_post_fwd(Cn, W, H, viewmats, render_colors, render_depths, render_alphas, render_normals, out_colors,
                    out_normals):
    a = make_args("gssdf_render_post_fwd_args", C=Cn, image_width=W, image_height=H, viewmats=viewmats,
                  render_colors=render_colors, render_depths=render_depths, render_alphas=render_alphas,
                  render_normals=render_normals, out_colors=out_colors, out_normals=out_normals)
    check(lib().gssdf_render_post_fwd(_lib.C.byref(a), _stream()))


def render_post_bwd(Cn, W, H, viewmats, render_depths, render_alphas, v_out_colors, v_out_normals, v_alphas_in,
                    v_render_colors, v_render_depths, v_render_alphas, v_render_normals):
    a = make_args("gssdf_render_post_bwd_args", C=Cn, image_width=W, image_height=H, viewmats=viewmats,
                  render_depths=render_depths, render_alphas=render_alphas, v_out_colors=v_out_colors,
                  v_out_normals=v_out_normals, v_alphas_in=v_alphas_in, v_render_colors=v_render_colors,
                  v_render_depths=v_render_depths, v_render_alphas=v_render_alphas, v_render_normals=v_render_normals)
    check(lib().gssdf_render_post_bwd(_lib.C.byref(a), _stream()))


def l1_loss(Cn, W, H, out_colors, gt, w_rgb, w_depth, loss_out, v_out_colors):
    a = make_args("gssdf_l1_loss_args", C=Cn, image_width=W, image_height=H, out_colors=out_colors, gt=gt, w_rgb=w_rgb,
                  w_depth=w_depth, loss_out=loss_out, v_out_colors=v_out_colors)
    check(lib().gssdf_l1_loss(_lib.C.byref(a), _stream()))


def render_post_bg_fwd(Cn, W, H, viewmats, render_colors, render_depths, render_alphas, render_normals, out_colors, out_normals,
                       bck_mode, bg=None):
    """render_post_fwd with the background composited into the colour: bck_mode 0 black, 1 white, 2 bg [C,H,W,3]."""
    post = make_args("gssdf_render_post_fwd_args", C=Cn, image_width=W, image_height=H, viewmats=viewmats,
                     render_colors=render_colors, render_depths=render_depths, render_alphas=render_alphas,
                     render_normals=render_normals, out_colors=out_colors, out_normals=out_normals)
    a = make_args("gssdf_render_post_bg_fwd_args", post=post, bck_mode=int(bck_mode), bg=bg)
    check(lib().gssdf_render_post_bg_fwd(_lib.C.byref(a), _stream()))


def render_post_bg_bwd(Cn, W, H, viewmats, render_depths, render_alphas, v_out_colors, v_out_normals, v_alphas_in,
                       v_render_colors, v_render_depths, v_render_alphas, v_render_normals, bck_mode, bg=None):
    post = make_args("gssdf_render_post_bwd_args", C=Cn, image_width=W, image_height=H, viewmats=viewmats,
                     render_depths=render_depths, render_alphas=render_alphas, v_out_colors=v_out_colors,
                     v_out_normals=v_out_normals, v_alphas_in=v_alphas_in, v_render_colors=v_render_colors,
                     v_render_depths=v_render_depths, v_render_alphas=v_render_alphas, v_render_normals=v_render_normals)
    a = make_args("gssdf_render_post_bg_bwd_args", post=post, bck_mode=int(bck_mode), bg=bg)
    check(lib().gssdf_render_post_bg_bwd(_lib.C.byref(a), _stream()))


def l1_loss_masked(Cn, W, H, out_colors, gt, w_rgb, w_depth, loss_out, v_out_colors, mask):
    """l1_loss with the rgb differences multiplied by mask (uint8 [H,W,3], nonzero = 1, shared by the C cameras)."""
    loss = make_args("gssdf_l1_loss_args", C=Cn, image_width=W, image_height=H, out_colors=out_colors, gt=gt, w_rgb=w_rgb,
                     w_depth=w_depth, loss_out=loss_out, v_out_colors=v_out_colors)
    a = make_args("gssdf_l1_loss_masked_args", loss=loss, mask=mask)
    check(lib().gssdf_l1_loss_masked(_lib.C.byref(a), _stream()))


def frames_u8_expand(store, offset, W, H, gt):
    """gt [H,W,4] (float32, contiguous) <- frame of W x H interleaved RGB bytes at byte `offset` of the uint8 CUDA tensor `store`, as
    x * (1.0f / 255.0f) in fp32; channel 3 <- 0 (gssdf_frames_u8_expand)."""
    _req(store, torch.uint8, "store")
    _req(gt, torch.float32, "gt")
    if offset < 0 or offset + 3 * W * H > store.numel() or gt.numel() < 4 * W * H:
        raise ValueError(f"gssdf_b200: a {W}x{H} frame at byte {offset} does not fit a store of {store.numel()} bytes and a gt of "
                         f"{gt.numel()} floats")
    a = make_args("gssdf_frames_u8_expand_args", store=store, offset=int(offset), W=W, H=H, gt=gt)
    check(lib().gssdf_frames_u8_expand(_lib.C.byref(a), _stream()))


def undistort_map(K, D, new_K, model, W, H, out):
    """out int16 [H,W,4] (CUDA, contiguous) <- the fixed-point undistortion map of one camera (gssdf_undistort_map). K, new_K: 3x3,
    D: up to 5 coefficients (k1 k2 p1 p2 k3 for model 0, k1..k4 for model 1); all are passed as fp32."""
    _req(out, torch.int16, "map")
    if out.numel() < 4 * W * H:
        raise ValueError(f"gssdf_b200: a map of {out.numel()} int16 is too small for {W}x{H}")
    d = [float(v) for v in torch.as_tensor(D, dtype=torch.float32).reshape(-1).tolist()]
    if len(d) > 5:
        raise ValueError(f"gssdf_b200: {len(d)} distortion coefficients, at most 5")
    f9 = lambda M: torch.as_tensor(M, dtype=torch.float32).reshape(-1).tolist()
    a = make_args("gssdf_undistort_map_args", model=int(model), W=int(W), H=int(H), K=f9(K), D=d + [0.0] * (5 - len(d)), new_K=f9(new_K),
                  map=out)
    check(lib().gssdf_undistort_map(_lib.C.byref(a), _stream()))


def undistort_u8(src, dst, offsets, sizes, map_ids, maps):
    """dst <- src remapped frame by frame (gssdf_undistort_u8). src, dst: uint8 CUDA tensors of one size holding packed RGB frames;
    offsets / sizes / map_ids: per-frame byte offsets, (W, H) and indices into `maps` (host sequences); maps: int16 [H,W,4] CUDA maps."""
    _req(src, torch.uint8, "src")
    _req(dst, torch.uint8, "dst")
    if src.numel() != dst.numel():
        raise ValueError(f"gssdf_b200: src has {src.numel()} bytes, dst {dst.numel()}")
    for m in maps:
        _req(m, torch.int16, "map")
        if m.device != src.device or dst.device != src.device:
            raise ValueError(f"gssdf_b200: src, dst and every map must be on one device ({src.device}, {dst.device}, {m.device})")
    n, C = len(offsets), _lib.C
    off = (C.c_int64 * max(n, 1))(*[int(o) for o in offsets])
    sz = (C.c_int32 * max(2 * n, 1))(*[int(v) for wh in sizes for v in wh])
    ids = (C.c_int32 * max(n, 1))(*[int(i) for i in map_ids])
    mp = (C.c_void_p * max(len(maps), 1))(*[m.data_ptr() for m in maps])
    msz = (C.c_int32 * max(2 * len(maps), 1))(*[v for m in maps for v in (int(m.shape[1]), int(m.shape[0]))])
    a = make_args("gssdf_undistort_u8_args", n_frames=n, n_bytes=src.numel(), src=src, dst=dst, offsets=C.addressof(off),
                  sizes=C.addressof(sz), map_ids=C.addressof(ids), n_maps=len(maps), maps=C.addressof(mp), map_sizes=C.addressof(msz))
    check(lib().gssdf_undistort_u8(_lib.C.byref(a), _stream()))


# ---- SDF branch -------------------------------------------------------------------------------
def sdf_net(table_half, mlp, n_levels=16, n_features=2, log2_hashmap_size=19, base_resolution=32, per_level_scale=2.0,
            hidden_dim=64, n_hidden=3, origin=(0.0, 0.0, 0.0), inv_size=0.0, mlp_mode=0, mlp_packed=None):
    """The struct holds RAW pointers: the caller keeps table_half / mlp / mlp_packed alive."""
    return make_args("gssdf_sdf_net", n_levels=n_levels, n_features_per_level=n_features, log2_hashmap_size=log2_hashmap_size,
                     base_resolution=base_resolution, per_level_scale=per_level_scale, hidden_dim=hidden_dim, n_hidden=n_hidden,
                     table_half=table_half, mlp=mlp, origin=list(origin), inv_size=inv_size, mlp_mode=mlp_mode,
                     mlp_packed=mlp_packed)


def sdf_table_params(net):
    return int(lib().gssdf_sdf_table_params(_lib.C.byref(net)))


def sdf_mlp_params(net):
    return int(lib().gssdf_sdf_mlp_params(_lib.C.byref(net)))


def sdf_mlp_packed_bytes(net):
    return int(lib().gssdf_sdf_mlp_packed_bytes(_lib.C.byref(net)))


def sdf_mlp_pack(net, packed):
    """Pre-split the hidden layers' weights (bf16 hi/mid/lo, operand layout) for mlp_mode=1; `packed` = uint8 device tensor."""
    assert packed.numel() * packed.element_size() >= sdf_mlp_packed_bytes(net)
    check(lib().gssdf_sdf_mlp_pack(_lib.C.byref(net), _lib.C.c_void_p(packed.data_ptr()), _stream()))


def sdf_table_to_half(table_f32, table_f16):
    check(lib().gssdf_sdf_table_to_half(_lib.C.c_void_p(table_f32.data_ptr()), _lib.C.c_void_p(table_f16.data_ptr()),
                                        _lib.C.c_int64(table_f32.numel()), _stream()))


def sdf_fwd(net, x, sdf, y1=None, feat=None, n_variants=1, delta=0.0, n_live=None, skip_base_variant=False):
    a = make_args("gssdf_sdf_fwd_args", n=x.shape[0], x=x, sdf=sdf, y1=y1, feat=feat, n_variants=n_variants, delta=delta, n_live=n_live,
                  skip_base_variant=int(bool(skip_base_variant)))
    a.net = net
    check(lib().gssdf_sdf_fwd(_lib.C.byref(a), _stream()))


def sdf_bwd(net, x, v_sdf, v_y1=None, table_grad=None, mlp_grad=None, v_x=None, n_variants=1, delta=0.0, n_live=None):
    a = make_args("gssdf_sdf_bwd_args", n=x.shape[0], x=x, v_sdf=v_sdf, v_y1=v_y1, table_grad=table_grad, mlp_grad=mlp_grad, v_x=v_x,
                  n_variants=n_variants, delta=delta, n_live=n_live)
    a.net = net
    check(lib().gssdf_sdf_bwd(_lib.C.byref(a), _stream()))


def sdf_loss(n, n_variants, sdf, y1, gt_sdf, weights, bce_isigma, bce_weight, eikonal_weight, gs_sdf_weight, delta, loss_out, v_sdf, v_y1,
             visibilities=None, visible_thr=0.0, n_live=None, valid_mask=None, n_gate=None):
    a = make_args("gssdf_sdf_loss_args", n=n, n_variants=n_variants, sdf=sdf, y1=y1, gt_sdf=gt_sdf, weights=weights,
                  visibilities=visibilities, visible_thr=visible_thr, n_live=n_live, valid_mask=valid_mask, n_gate=n_gate,
                  bce_isigma=bce_isigma, bce_weight=bce_weight, eikonal_weight=eikonal_weight, gs_sdf_weight=gs_sdf_weight,
                  delta=delta, loss_out=loss_out, v_sdf=v_sdf, v_y1=v_y1)
    check(lib().gssdf_sdf_loss(_lib.C.byref(a), _stream()))


def sdf_train(net, x, n_variants, delta, gt_sdf, weights, bce_isigma, bce_weight, eikonal_weight, gs_sdf_weight, loss_out,
              table_grad=None, mlp_grad=None, v_x=None, visibilities=None, visible_thr=0.0, n_live=None, eikonal_mode=0,
              align_weight=0.0, sdf_variants=None, valid_mask=None, n_gate=None):
    """sdf_fwd + sdf_loss + sdf_bwd fused into one persistent tensor-core kernel (net.mlp_mode must be 1)."""
    a = make_args("gssdf_sdf_train_args", n=x.shape[0], x=x, n_variants=n_variants, delta=delta, n_live=n_live, gt_sdf=gt_sdf,
                  weights=weights, visibilities=visibilities, visible_thr=visible_thr, bce_isigma=bce_isigma, bce_weight=bce_weight,
                  eikonal_weight=eikonal_weight, gs_sdf_weight=gs_sdf_weight, loss_out=loss_out, table_grad=table_grad,
                  mlp_grad=mlp_grad, v_x=v_x, eikonal_mode=eikonal_mode, align_weight=align_weight,
                  sdf_variants=sdf_variants, valid_mask=valid_mask, n_gate=n_gate)
    a.net = net
    check(lib().gssdf_sdf_train(_lib.C.byref(a), _stream()))


def dssim_loss(Cn, W, H, out_colors, gt, w_dssim, loss_out, v_out_colors, ws):
    """loss_out += w_dssim * (1 - SSIM(rgb, gt_rgb)); v_out_colors[..., :3] += gradient (call after l1_loss)."""
    need = lib().gssdf_dssim_workspace_bytes(Cn, W, H)
    w = ws.get(need)
    a = make_args("gssdf_dssim_loss_args", C=Cn, image_width=W, image_height=H, out_colors=out_colors, gt=gt, w_dssim=w_dssim,
                  loss_out=loss_out, v_out_colors=v_out_colors, workspace=w, workspace_bytes=w.numel())
    check(lib().gssdf_dssim_loss(_lib.C.byref(a), _stream()))


def dssim_loss_masked(Cn, W, H, out_colors, gt, w_dssim, loss_out, v_out_colors, ws, mask):
    """dssim_loss of rgb * mask against gt * mask (mask uint8 [H,W,3], nonzero = 1); the gradient is masked too."""
    need = lib().gssdf_dssim_workspace_bytes(Cn, W, H)
    w = ws.get(need)
    loss = make_args("gssdf_dssim_loss_args", C=Cn, image_width=W, image_height=H, out_colors=out_colors, gt=gt, w_dssim=w_dssim,
                     loss_out=loss_out, v_out_colors=v_out_colors, workspace=w, workspace_bytes=w.numel())
    a = make_args("gssdf_dssim_loss_masked_args", loss=loss, mask=mask)
    check(lib().gssdf_dssim_loss_masked(_lib.C.byref(a), _stream()))


# ---- operator-level hash grid (tcnn_binding twin), gate, optimiser, remaining loss terms ------------------------------------
def hashgrid_fwd(net, x, feat):
    a = make_args("gssdf_hashgrid_fwd_args", n=x.shape[0], x=x, feat=feat)
    a.net = net
    check(lib().gssdf_hashgrid_fwd(_lib.C.byref(a), _stream()))


def hashgrid_bwd(net, x, dL_dy, table_grad=None, dL_dx=None):
    a = make_args("gssdf_hashgrid_bwd_args", n=x.shape[0], x=x, dL_dy=dL_dy, table_grad=table_grad, dL_dx=dL_dx)
    a.net = net
    check(lib().gssdf_hashgrid_bwd(_lib.C.byref(a), _stream()))


def hashgrid_bwdbwd(net, x, dL_ddLdx, dL_dy, table_grad=None, dL_ddLdy=None, dL_dx=None):
    a = make_args("gssdf_hashgrid_bwdbwd_args", n=x.shape[0], x=x, dL_ddLdx=dL_ddLdx, dL_dy=dL_dy, table_grad=table_grad,
                  dL_ddLdy=dL_ddLdy, dL_dx=dL_dx)
    a.net = net
    check(lib().gssdf_hashgrid_bwdbwd(_lib.C.byref(a), _stream()))


def sdf_gate_count(n, n_gate, visibilities=None, visible_thr=0.0, valid_mask=None, n_live=None):
    a = make_args("gssdf_sdf_gate_count_args", n=n, n_live=n_live, visibilities=visibilities, visible_thr=visible_thr,
                  valid_mask=valid_mask, n_gate=n_gate)
    check(lib().gssdf_sdf_gate_count(_lib.C.byref(a), _stream()))


def normal_consistency_loss(Cn, W, H, viewmats, Ks, depth, depth_stride, render_alphas, out_normals, weight, loss_out, v_depth=None,
                            v_depth_stride=1, v_out_normals=None):
    """depth / v_depth are raw device pointers (int) or tensors: e.g. out_colors.data_ptr() + 12 with stride 4 for the ED channel."""
    a = make_args("gssdf_normal_consistency_args", C=Cn, image_width=W, image_height=H, viewmats=viewmats, Ks=Ks, depth=depth,
                  depth_stride=depth_stride, render_alphas=render_alphas, out_normals=out_normals, weight=weight, loss_out=loss_out,
                  v_depth=v_depth, v_depth_stride=v_depth_stride, v_out_normals=v_out_normals)
    check(lib().gssdf_normal_consistency_loss(_lib.C.byref(a), _stream()))


def isotropic_loss(N, cap, counts, gaussian_ids, scales, raw_params, weight, loss_out, v_scales=None):
    a = make_args("gssdf_isotropic_loss_args", N=N, cap=cap, counts=counts, gaussian_ids=gaussian_ids, scales=scales,
                  raw_params=int(bool(raw_params)), weight=weight, loss_out=loss_out, v_scales=v_scales)
    check(lib().gssdf_isotropic_loss(_lib.C.byref(a), _stream()))


ADAM_WINDOW = 64  # GSSDF_ADAM_WINDOW


class AdamReplay:
    """Host half of the lazy row groups (gssdf_adam_replay): the device stamps `last` [rows] (int32) and the scalars of the last
    ADAM_WINDOW steps. push(t, lr0, lr1) once per step, before that step's adam_step."""

    def __init__(self, last, beta1=0.9, beta2=0.999, eps=1e-15):
        self.last = last
        self.s = make_args("gssdf_adam_replay", last=last, beta1=beta1, beta2=beta2, eps=eps)

    def push(self, step, lr0, lr1):
        check(lib().gssdf_adam_replay_push(_lib.C.byref(self.s), int(step), float(lr0), float(lr1)))

    @property
    def step(self):
        return self.s.step

    def ptr(self):
        return _lib.C.addressof(self.s)


def _adam_args(params, grads, exp_avg, exp_avg_sq, groups, step, beta1=0.9, beta2=0.999, eps=1e-15, grad_scale=1.0, zero_grads=True,
               table_half=None, net=None, mlp_packed=None, replay=None, row_ids=None, row_count=None, row_cap=0, replay_only=False):
    a = make_args("gssdf_adam_args", params=params, grads=grads, exp_avg=exp_avg, exp_avg_sq=exp_avg_sq, n_groups=len(groups), step=step,
                  beta1=beta1, beta2=beta2, eps=eps, grad_scale=grad_scale, zero_grads=int(bool(zero_grads)), table_half=table_half,
                  mlp_packed=mlp_packed, replay=replay.ptr() if replay is not None else None, row_ids=row_ids, row_count=row_count,
                  row_cap=int(row_cap), replay_only=int(bool(replay_only)))
    for i, grp in enumerate(groups):
        off, cnt, lr, hs = grp[:4]
        a.groups[i].offset, a.groups[i].count, a.groups[i].lr, a.groups[i].half_shadow = int(off), int(cnt), float(lr), int(bool(hs))
        a.groups[i].row_width = int(grp[4]) if len(grp) > 4 else 0
    if net is not None:
        a.net = _lib.C.cast(_lib.C.pointer(net), _lib.C.c_void_p)
    return a


def adam_step(params, grads, exp_avg, exp_avg_sq, groups, step, **kw):
    """groups: list of (offset, count, lr, half_shadow[, row_width]). `net` (gssdf_sdf_net struct, kept alive by the caller) + mlp_packed:
    re-pack the decoder's bf16 operand image after the update. Row groups (row_width > 0) need `replay` (AdamReplay, pushed for `step`);
    row_ids + row_count (device counts, ->nnz) + row_cap: visit those rows only, else every row (see gssdf_adam_args). Keywords: beta1,
    beta2, eps, grad_scale, zero_grads, table_half, net, mlp_packed, replay, row_ids, row_count, row_cap, replay_only."""
    check(lib().gssdf_adam_step(_lib.C.byref(_adam_args(params, grads, exp_avg, exp_avg_sq, groups, step, **kw)), _stream()))


def adam_step_clocks(params, grads, exp_avg, exp_avg_sq, groups, steps, **kw):
    """adam_step with one step per group (`steps`, a sequence as long as `groups`; the row groups share one step, for which `replay` is
    pushed): gssdf_adam_step_clocks."""
    if len(steps) != len(groups):
        raise ValueError(f"gssdf_b200: {len(steps)} steps for {len(groups)} groups")
    a = _adam_args(params, grads, exp_avg, exp_avg_sq, groups, 1, **kw)
    st = (_lib.C.c_int32 * max(len(steps), 1))(*[int(t) for t in steps])
    check(lib().gssdf_adam_step_clocks(_lib.C.byref(a), _lib.C.cast(st, _lib.C.c_void_p), _stream()))


def _rows_args(segments, cap_rows, n_rows, row_ids, flat, packed, zero_source=False):
    a = make_args("gssdf_rows_args", n_segments=len(segments), zero_source=int(bool(zero_source)), cap_rows=cap_rows, n_rows=n_rows,
                  row_ids=row_ids, flat=flat, packed=packed)
    for i, (off, width) in enumerate(segments):
        a.segments[i].offset, a.segments[i].width = int(off), int(width)
    return a


def rows_stride(segments):
    return 1 + sum(int(w) for _, w in segments)


def rows_pack(segments, cap_rows, n_rows, row_ids, flat, packed, zero_source=False):
    """segments: list of (offset, width) into `flat`. packed[k] = [id | flat rows row_ids[k] of every segment], k < *n_rows (device int32);
    zero_source: the packed elements of `flat` are cleared."""
    check(lib().gssdf_rows_pack(_lib.C.byref(_rows_args(segments, cap_rows, n_rows, row_ids, flat, packed, zero_source)), _stream()))


def rows_unpack_add(segments, cap_rows, n_rows, flat, packed):
    """flat rows += packed rows (the ids travel in column 0 of the packed rows)."""
    check(lib().gssdf_rows_unpack_add(_lib.C.byref(_rows_args(segments, cap_rows, n_rows, None, flat, packed)), _stream()))


def sdf_gate_compact(n, x, index, x_out, n_gate, ws, visibilities=None, visible_thr=0.0, valid_mask=None, weights=None, w_out=None, n_live=None):
    """Stable compaction of the samples passing `vis > thr & valid` (the reference's index_select, neural_mapping.cpp:433-437)."""
    w = ws.get(lib().gssdf_sdf_gate_compact_workspace_bytes(_lib.C.c_int64(n)))
    a = make_args("gssdf_sdf_gate_compact_args", n=n, n_live=n_live, visibilities=visibilities, visible_thr=visible_thr, valid_mask=valid_mask,
                  x=x, weights=weights, index=index, x_out=x_out, w_out=w_out, n_gate=n_gate, workspace=w, workspace_bytes=w.numel())
    check(lib().gssdf_sdf_gate_compact(_lib.C.byref(a), _stream()))


def sdf_outlier_filter(net, xyz, threshold, columns, n_kept, ws, index=None, n=None):
    """Rows r < n (default: all of xyz) with |sdf(xyz[r])| < threshold (fp32), in order: index[j] = j-th kept row (or None), *n_kept = count
    (device int64 [1]), and for each (src, dst) of `columns` (contiguous CUDA tensors of equal row width) dst[j] = src[index[j]]."""
    n = xyz.shape[0] if n is None else int(n)
    w = ws.get(lib().gssdf_sdf_outlier_filter_workspace_bytes(_lib.C.c_int64(n)))
    a = make_args("gssdf_sdf_outlier_filter_args", n=n, xyz=_req(xyz, torch.float32, "xyz"), threshold=threshold, n_columns=len(columns),
                  index=_req(index, torch.int64, "index"), n_kept=_req(n_kept, torch.int64, "n_kept"), workspace=w, workspace_bytes=w.numel())
    a.net = net
    for i, (src, dst) in enumerate(columns[:len(a.columns)]):  # more columns than the struct holds: n_columns makes the library refuse
        for name, t in (("src", src), ("dst", dst)):
            if not (t.is_cuda and t.is_contiguous()):
                raise ValueError(f"gssdf_b200: column {i} {name} must be a contiguous CUDA tensor")
        a.columns[i].src, a.columns[i].dst = src.data_ptr() or None, dst.data_ptr() or None
        a.columns[i].row_bytes = math.prod(src.shape[1:]) * src.element_size()
    check(lib().gssdf_sdf_outlier_filter(_lib.C.byref(a), _stream()))


def sdf_fwd_dev(net, x, sdf, delta, y1=None, feat=None, n_variants=1, n_live=None, skip_base_variant=False):
    """sdf_fwd with the offset read from the device: delta = float32 CUDA tensor [1]."""
    a = make_args("gssdf_sdf_fwd_args", n=x.shape[0], x=x, sdf=sdf, y1=y1, feat=feat, n_variants=n_variants, n_live=n_live,
                  skip_base_variant=int(bool(skip_base_variant)))
    a.net = net
    check(lib().gssdf_sdf_fwd_dev(_lib.C.byref(a), _lib.C.c_void_p(_req(delta, torch.float32, "delta").data_ptr()), _stream()))


def sdf_train_dev(net, x, n_variants, delta, gt_sdf, weights, bce_isigma, bce_weight, eikonal_weight, gs_sdf_weight, loss_out,
                  table_grad=None, mlp_grad=None, v_x=None, visibilities=None, visible_thr=0.0, n_live=None, eikonal_mode=0,
                  align_weight=0.0, sdf_variants=None, valid_mask=None, n_gate=None):
    """sdf_train with the offset read from the device: delta = float32 CUDA tensor [1]."""
    a = make_args("gssdf_sdf_train_args", n=x.shape[0], x=x, n_variants=n_variants, n_live=n_live, gt_sdf=gt_sdf,
                  weights=weights, visibilities=visibilities, visible_thr=visible_thr, bce_isigma=bce_isigma, bce_weight=bce_weight,
                  eikonal_weight=eikonal_weight, gs_sdf_weight=gs_sdf_weight, loss_out=loss_out, table_grad=table_grad,
                  mlp_grad=mlp_grad, v_x=v_x, eikonal_mode=eikonal_mode, align_weight=align_weight,
                  sdf_variants=sdf_variants, valid_mask=valid_mask, n_gate=n_gate)
    a.net = net
    check(lib().gssdf_sdf_train_dev(_lib.C.byref(a), _lib.C.c_void_p(_req(delta, torch.float32, "delta").data_ptr()), _stream()))


def sdf_sample_rays_dev(args, n_rays_live=None, sample_std=None):
    """gssdf_sdf_sample_rays on a filled gssdf_sdf_sample_rays_args (octree.RaySampler builds it) with a device ray count (int32 [1])
    and a device std (float32 [1]); args.n_rays is the capacity."""
    nl = _req(n_rays_live, torch.int32, "n_rays_live")
    sd = _req(sample_std, torch.float32, "sample_std")
    check(lib().gssdf_sdf_sample_rays_dev(_lib.C.byref(args), _lib.C.c_void_p(nl.data_ptr() if nl is not None else None),
                                          _lib.C.c_void_p(sd.data_ptr() if sd is not None else None), _stream()))


def sdf_ray_batch(pack, rand, n_rays, out, index=None):
    """Rows i < *n_rays of out = pack rows clamp((int64)(rand[i] * (float)N), 0, N - 1). pack / out: dicts of contiguous CUDA float32
    origin [.,3], direction [.,3], depth [.] or [.,1], xyz [.,3]; N = pack rows, ray capacity = rand.numel(); n_rays: int32 CUDA [1]."""
    N = pack["xyz"].shape[0]
    f32 = torch.float32
    a = make_args("gssdf_sdf_ray_batch_args", N=N, ray_cap=rand.numel(), rand=_req(rand, f32, "rand"),
                  n_rays=_req(n_rays, torch.int32, "n_rays"), index=_req(index, torch.int64, "index"),
                  **{k: _req(pack[k], f32, k) for k in ("origin", "direction", "depth", "xyz")},
                  **{k + "_out": _req(out[k], f32, k + "_out") for k in ("origin", "direction", "depth", "xyz")})
    check(lib().gssdf_sdf_ray_batch(_lib.C.byref(a), _stream()))


def sdf_adapt(state, y1, n_samples, bce_sigma, bce_isigma, batch_pt_num, update_rays=True):
    """One nsdf_train / sdf_train_callback state update on the device. state: int32 CUDA [4] holding gssdf_sdf_adapt_state
    {float sample_std, float pts_per_ray, int32 n_rays, pad} (see nsdf.new_adapt_state); y1: float32 [cap] (variant-0 rows);
    n_samples: int32 CUDA tensor whose first element is the sample count."""
    a = make_args("gssdf_sdf_adapt_args", state=_req(state, state.dtype, "state"), y1=_req(y1, torch.float32, "y1"), y1_cap=y1.numel(),
                  n_samples=_req(n_samples, torch.int32, "n_samples"), bce_sigma=bce_sigma, bce_isigma=bce_isigma,
                  batch_pt_num=batch_pt_num, update_rays=int(bool(update_rays)))
    check(lib().gssdf_sdf_adapt(_lib.C.byref(a), _stream()))


def scatter_rows3(n, index, n_gate, src, dst, n_live=None):
    a = make_args("gssdf_scatter_rows3_args", n=n, n_live=n_live, index=index, n_gate=n_gate, src=src, dst=dst)
    check(lib().gssdf_scatter_rows3(_lib.C.byref(a), _stream()))


def densify_update_state(N, cap, counts, gaussian_ids, v_densify, visibilities, radii, width, height, n_cameras, grad2d, count, vis, radii_state=None,
                         image_size=None):
    """image_size: the radii normaliser (gssdf_densify_update_state_sized); None: max(width, height) of this call
    (gssdf_densify_update_state). grad2d scales by this call's width and height either way."""
    a = make_args("gssdf_densify_update_args", N=N, cap=cap, counts=counts, gaussian_ids=gaussian_ids, v_densify=v_densify, visibilities=visibilities,
                  radii=radii, width=width, height=height, n_cameras=n_cameras, grad2d=grad2d, count=count, vis=vis, radii_state=radii_state)
    if image_size is None:
        check(lib().gssdf_densify_update_state(_lib.C.byref(a), _stream()))
    else:
        check(lib().gssdf_densify_update_state_sized(_lib.C.byref(a), _lib.C.c_float(image_size), _stream()))


def densify_flags(N, offsets, quats, scaling, opacity, flags, grad2d=None, count=None, vis=None, radii_state=None, grow_grad2d=0.0, grow_scale3d=0.0,
                  grow_scale2d=0.0, use_scale2d=False, prune_opa=0.0, prune_scale3d=float("inf")):
    a = make_args("gssdf_densify_flags_args", N=N, offsets=offsets, quats=quats, scaling=scaling, opacity=opacity, grad2d=grad2d, count=count, vis=vis,
                  radii_state=radii_state, grow_grad2d=grow_grad2d, grow_scale3d=grow_scale3d, grow_scale2d=grow_scale2d, use_scale2d=int(bool(use_scale2d)),
                  prune_opa=prune_opa, prune_scale3d=prune_scale3d, flags=flags)
    check(lib().gssdf_densify_flags(_lib.C.byref(a), _stream()))


def densify_remap(n_new, K, stride_old, stride_new, src_row, mode, randn_row, randn, old, new, states_old=(), states_new=()):
    """old / new: dict(params, exp_avg, exp_avg_sq, anchors)."""
    a = make_args("gssdf_densify_remap_args", n_new=n_new, K=K, stride_old=stride_old, stride_new=stride_new, src_row=src_row, mode=mode,
                  randn_row=randn_row, randn=randn, params_old=old["params"], exp_avg_old=old["exp_avg"], exp_avg_sq_old=old["exp_avg_sq"],
                  anchors_old=old["anchors"], params_new=new["params"], exp_avg_new=new["exp_avg"], exp_avg_sq_new=new["exp_avg_sq"],
                  anchors_new=new["anchors"], n_state=len(states_old))
    for i, (so, sn) in enumerate(zip(states_old, states_new)):
        a.state_old[i], a.state_new[i] = so.data_ptr(), sn.data_ptr()
    check(lib().gssdf_densify_remap(_lib.C.byref(a), _stream()))


def l2_persist(tensor, hit_ratio=1.0):
    """Keep `tensor` (e.g. the fp16 hash-table shadow) resident in L2 for kernels launched on the current stream (None clears the window)."""
    if tensor is None:
        check(lib().gssdf_l2_persist(None, 0, 1.0, _stream()))
    else:
        check(lib().gssdf_l2_persist(_lib.C.c_void_p(tensor.data_ptr()), tensor.numel() * tensor.element_size(), hit_ratio, _stream()))
