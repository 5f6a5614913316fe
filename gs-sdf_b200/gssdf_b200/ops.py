"""Host-side mirror of the reference operator surface for the splat path.

Same names, argument meaning, return arity and error behaviour as the reference's libtorch wrappers
(GSC = /root/reference/submodules/gsplat_cpp/gsplat_cpp):
  fully_fused_projection_2dgs   GSC/fully_fused_projection.h:53-63  (.cpp:171-310)
  get_view_colors               GSC/rendering.h:8-13               (.cpp:11-47)
  isect_tiles / isect_offset_encode / tile_encode
                                GSC/isect_tiles.hpp:8-46, GSC/rendering.h:15-20 (.cpp:49-63)
  rasterize_to_pixels_2dgs      GSC/rasterize_to_pixels.h:64-80    (.cpp:170-381)
  rasterization_2dgs_sdf        include/neural_gaussian/neural_gaussian.cpp:129-271
All compute happens in libgssdf_b200.so (hand-written sm_90a CUDA) through gssdf_b200.cabi; torch is
used for device memory, streams and autograd plumbing only. The C++/libtorch twin of this file, meant
to be linked into neural_mapping_node, is gs-sdf_b200/shim/.

The functions here return exactly-shaped tensors ([nnz, ...], [n_isects]) like the reference, which costs
ONE host read-back of the two device counters per render (the reference blocks three times). The fully
asynchronous, capacity-based path used for throughput is gssdf_b200.render.SplatRenderer.
"""
import math

import torch

from . import cabi

_WS = {}


def _ws(device):
    key = (device.type, device.index)
    if key not in _WS:
        _WS[key] = cabi.Workspace(device)
    return _WS[key]


def _check(cond, msg):
    if not cond:
        raise ValueError(msg)  # TORCH_CHECK -> c10::Error in the reference


class _Packed:
    """Device counters + capacity that travel with the packed tensors of one render."""

    def __init__(self, counts, cap):
        self.counts, self.cap = counts, cap


# ----------------------------------------------------------------------------------------------
# projection
# ----------------------------------------------------------------------------------------------
class FullyFusedProjectionPacked2DGS(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means, quats, scales, viewmats, Ks, width, height, near_plane, far_plane, radius_clip, sparse_grad,
                randns):
        N, C = means.shape[0], viewmats.shape[0]
        dev = means.device
        cap = N * C
        f32 = dict(dtype=torch.float32, device=dev)
        out = dict(camera_ids=torch.empty(cap, dtype=torch.int64, device=dev),
                   gaussian_ids=torch.empty(cap, dtype=torch.int64, device=dev),
                   radii=torch.empty(cap, 2, dtype=torch.int32, device=dev), means2d=torch.empty(cap, 2, **f32),
                   depths=torch.empty(cap, **f32), ray_transforms=torch.empty(cap, 3, 3, **f32),
                   normals=torch.empty(cap, 3, **f32), samples=torch.empty(cap, 3, **f32),
                   sample_weights=torch.empty(cap, 1, **f32), indptr=torch.empty(C + 1, dtype=torch.int32, device=dev))
        counts = cabi.new_counts(dev)
        if randns is None:
            # the reference draws at::randn({nnz,2}) after its sync (Projection.cpp:728); we draw the
            # capacity up front from the same ATen generator so the call stays asynchronous
            randns = torch.randn(cap, 2, **f32)
        cabi.project2dgs_fwd(means, quats, scales, viewmats, Ks, width, height, near_plane, far_plane, radius_clip, randns,
                             cap, out, counts, _ws(dev))
        nnz = int(counts[cabi.NNZ].item())  # the one host read-back of the exact-shape API
        ctx.save_for_backward(out["camera_ids"], out["gaussian_ids"], means, quats, scales, viewmats, Ks,
                              out["ray_transforms"], randns, counts)
        ctx.dims = (width, height, cap, nnz)
        ctx.mark_non_differentiable(out["camera_ids"], out["gaussian_ids"], out["radii"])
        pk = lambda k: out[k][:nnz]
        res = (pk("camera_ids"), pk("gaussian_ids"), pk("radii"), pk("means2d"), pk("depths"), pk("ray_transforms"),
               pk("normals"), pk("samples"), pk("sample_weights"))
        ctx.mark_non_differentiable(res[0], res[1], res[2])
        return res

    @staticmethod
    def backward(ctx, _vc, _vg, _vr, v_means2d, v_depths, v_ray_transforms, v_normals, v_samples, _vw):
        camera_ids, gaussian_ids, means, quats, scales, viewmats, Ks, ray_transforms, randns, counts = ctx.saved_tensors
        width, height, cap, nnz = ctx.dims
        c = lambda t: None if t is None else t.contiguous()
        v_means, v_quats, v_scales = torch.zeros_like(means), torch.zeros_like(quats), torch.zeros_like(scales)
        if nnz > 0:
            cabi.project2dgs_bwd(means, quats, scales, viewmats, Ks, width, height, nnz, counts, camera_ids, gaussian_ids,
                                 ray_transforms, randns, c(v_means2d), c(v_depths), c(v_ray_transforms), c(v_normals),
                                 c(v_samples), v_means, v_quats, v_scales)
        return (v_means, v_quats, v_scales) + (None,) * 9


def fully_fused_projection_2dgs(means, quats, scales, viewmats, Ks, width, height, near_plane=0.01, far_plane=1e10,
                                radius_clip=0.0, packed=False, sparse_grad=False, randns=None):
    """-> (camera_ids, gaussian_ids, radii, means2d, depths, ray_transforms, normals, samples, samples_weights).
    `randns` ([C*N,2], optional) pins the stochastic sample for parity tests."""
    C, N = viewmats.shape[0], means.shape[0]
    _check(tuple(means.shape) == (N, 3), "Invalid means size")
    _check(tuple(viewmats.shape) == (C, 4, 4), "Invalid viewmats size")
    _check(tuple(Ks.shape) == (C, 3, 3), "Invalid Ks size")
    _check(tuple(quats.shape) == (N, 4), "Invalid quats size")
    _check(tuple(scales.shape) == (N, 3), f"Invalid scales size: {tuple(scales.shape)}")
    _check(packed, "gssdf_b200 implements the packed 2DGS projection only (GS-SDF always passes packed=true)")
    _check(not sparse_grad, "sparse_grad is outside the GS-SDF path")
    return FullyFusedProjectionPacked2DGS.apply(means.contiguous(), quats.contiguous(), scales.contiguous(),
                                                viewmats.contiguous(), Ks.contiguous(), width, height, near_plane, far_plane,
                                                radius_clip, sparse_grad, randns)


# ----------------------------------------------------------------------------------------------
# view-dependent colour
# ----------------------------------------------------------------------------------------------
class _ViewColors(torch.autograd.Function):
    @staticmethod
    def forward(ctx, viewmats, means, radii, sh, camera_ids, gaussian_ids, sh_degree):
        nnz = gaussian_ids.shape[0]
        dev = means.device
        colors = torch.empty(nnz, 3, dtype=torch.float32, device=dev)
        counts = cabi.new_counts(dev, nnz=nnz)
        if nnz > 0:
            cabi.view_colors_fwd(viewmats, means, sh, sh_degree, nnz, counts, camera_ids, gaussian_ids, radii, colors)
        ctx.save_for_backward(viewmats, means, radii, sh, camera_ids, gaussian_ids, colors, counts)
        ctx.sh_degree = sh_degree
        return colors

    @staticmethod
    def backward(ctx, v_colors):
        viewmats, means, radii, sh, camera_ids, gaussian_ids, colors, counts = ctx.saved_tensors
        v_sh = torch.zeros_like(sh)
        v_means = torch.zeros_like(means) if ctx.needs_input_grad[1] else None
        nnz = gaussian_ids.shape[0]
        if nnz > 0:
            cabi.view_colors_bwd(viewmats, means, sh, ctx.sh_degree, nnz, counts, camera_ids, gaussian_ids, radii, colors,
                                 v_colors.contiguous(), v_sh, v_means)
        return None, v_means, None, v_sh, None, None, None


def get_view_colors(viewmats, means, radii, colors, camera_ids, gaussian_ids, sh_degree=None):
    """GSC/rendering.cpp:11-47. With sh_degree=None colours are gathered as in the reference (pure indexing)."""
    if sh_degree is None:
        return colors[gaussian_ids] if colors.dim() == 2 else colors[camera_ids, gaussian_ids]
    _check(colors.dim() == 3 and colors.shape[2] == 3, "Invalid colors shape")
    _check((sh_degree + 1) ** 2 <= colors.shape[1], "Invalid coeffs shape")
    return _ViewColors.apply(viewmats.contiguous(), means.contiguous(), radii.contiguous(), colors.contiguous(),
                             camera_ids.contiguous(), gaussian_ids.contiguous(), sh_degree)


# ----------------------------------------------------------------------------------------------
# tiles
# ----------------------------------------------------------------------------------------------
@torch.no_grad()
def _tile_encode_full(means2d, radii, depths, tile_size, tile_width, tile_height, n_cameras, camera_ids, image_wh=None):
    nnz = means2d.shape[0]
    _check(tuple(means2d.shape) == (nnz, 2), "Invalid shape for means2d")
    _check(tuple(radii.shape) == (nnz, 2), f"Invalid shape for radii: {tuple(radii.shape)}")
    _check(tuple(depths.shape) == (nnz,), "Invalid shape for depths")
    _check(camera_ids is not None, "camera_ids is required if packed is True")
    _check(n_cameras > 0, "n_cameras is required if packed is True")
    dev = means2d.device
    W, H = image_wh if image_wh is not None else (tile_width * tile_size, tile_height * tile_size)
    counts = cabi.new_counts(dev, nnz=nnz)
    tpg = torch.empty(nnz, dtype=torch.int32, device=dev)
    offsets = torch.empty(n_cameras, tile_height, tile_width, dtype=torch.int32, device=dev)
    # exact n_isects first (count-only call with zero capacity), then the real call: exact-shape API
    dummy = torch.empty(1, dtype=torch.int32, device=dev)
    cabi.tile_encode(n_cameras, W, H, tile_size, nnz, counts, means2d.contiguous(), radii.contiguous(), depths.contiguous(),
                     camera_ids.contiguous(), 0, tpg, None, dummy, offsets, _ws(dev))
    n_isects = int(tpg.sum(dtype=torch.int64).item()) if nnz > 0 else 0
    isect_ids = torch.empty(n_isects, dtype=torch.int64, device=dev)
    flatten_ids = torch.empty(max(n_isects, 1), dtype=torch.int32, device=dev)
    cabi.tile_encode(n_cameras, W, H, tile_size, nnz, counts, means2d.contiguous(), radii.contiguous(), depths.contiguous(),
                     camera_ids.contiguous(), n_isects, tpg, isect_ids, flatten_ids, offsets, _ws(dev))
    return tpg, isect_ids, flatten_ids[:n_isects], offsets


def isect_tiles(means2d, radii, depths, tile_size, tile_width, tile_height, sort=True, packed=False, n_cameras=-1,
                camera_ids=None, gaussian_ids=None):
    """GSC/isect_tiles.hpp:8-37 -> (tiles_per_gauss, isect_ids, flatten_ids); always sorted."""
    _check(packed, "gssdf_b200 implements the packed layout only")
    _check(sort, "unsorted intersections are never requested by GS-SDF")
    tpg, ids, flat, _ = _tile_encode_full(means2d, radii, depths, tile_size, tile_width, tile_height, n_cameras, camera_ids)
    return tpg, ids, flat


def tile_encode(width, height, tile_size, means2d, radii, depths, packed, camera_num, camera_ids, gaussian_ids=None):
    """GSC/rendering.cpp:49-63. Returns (isect_offsets, flatten_ids, isect_offsets) -- the first slot is NOT
    tiles_per_gauss; the reference has the same quirk (rendering.cpp:62)."""
    tw, th = int(math.ceil(width / float(tile_size))), int(math.ceil(height / float(tile_size)))
    _, _, flat, offsets = _tile_encode_full(means2d, radii, depths, tile_size, tw, th, camera_num, camera_ids,
                                            image_wh=(width, height))
    return offsets, flat, offsets


# ----------------------------------------------------------------------------------------------
# rasterisation
# ----------------------------------------------------------------------------------------------
class RasterizeToPixels2DGS(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means2d, ray_transforms, colors, opacities, normals, densify, backgrounds, masks, width, height,
                tile_size, isect_offsets, flatten_ids, absgrad, distloss):
        dev = means2d.device
        C = isect_offsets.shape[0]
        nnz = means2d.shape[0]
        n_isects = flatten_ids.shape[0]
        f32 = dict(dtype=torch.float32, device=dev)
        i32 = dict(dtype=torch.int32, device=dev)
        out = dict(render_colors=torch.empty(C, height, width, 3, **f32), render_depths=torch.empty(C, height, width, 1, **f32),
                   render_alphas=torch.empty(C, height, width, 1, **f32), render_normals=torch.empty(C, height, width, 3, **f32),
                   render_distort=torch.empty(C, height, width, 1, **f32), render_median=torch.empty(C, height, width, 1, **f32),
                   render_Ts=torch.empty(C, height, width, 2, **f32), last_ids=torch.empty(C, height, width, **i32),
                   median_ids=torch.empty(C, height, width, **i32), visibilities=torch.zeros(max(nnz, 1), 1, **f32))
        counts = cabi.new_counts(dev, nnz=nnz, n_isects=n_isects)
        cabi.raster2dgs_fwd(C, width, height, tile_size, colors.shape[-1], nnz, counts, means2d, ray_transforms, colors,
                            opacities, normals, backgrounds, isect_offsets, flatten_ids, out, _ws(dev))
        ctx.save_for_backward(means2d, ray_transforms, colors, opacities, normals, isect_offsets, flatten_ids,
                              out["render_alphas"], out["render_Ts"], out["last_ids"], out["median_ids"], counts,
                              backgrounds if backgrounds is not None else torch.empty(0, device=dev))
        ctx.dims = (width, height, tile_size, C, nnz, backgrounds is not None, absgrad is not None and absgrad.requires_grad)
        vis = out["visibilities"][:nnz]
        ctx.mark_non_differentiable(vis)
        return (out["render_colors"], out["render_depths"], out["render_alphas"], out["render_normals"],
                out["render_distort"], out["render_median"], vis)

    @staticmethod
    def backward(ctx, v_colors, v_depths, v_alphas, v_normals, v_distort, v_median, _v_vis):
        (means2d, ray_transforms, colors, opacities, normals, isect_offsets, flatten_ids, render_alphas, render_Ts,
         last_ids, median_ids, counts, bg) = ctx.saved_tensors
        width, height, tile_size, C, nnz, has_bg, want_abs = ctx.dims
        dev = means2d.device
        f32 = dict(dtype=torch.float32, device=dev)
        z = lambda t, *s: torch.zeros(*s, **f32) if t is None else t.contiguous()
        v_colors = z(v_colors, C, height, width, 3)
        v_depths = z(v_depths, C, height, width, 1)
        v_alphas = z(v_alphas, C, height, width, 1)
        v_normals = z(v_normals, C, height, width, 3)
        v_median = z(v_median, C, height, width, 1)
        # v_distort: GS-SDF passes distloss=false, so autograd materialises zeros here; the distortion
        # VJP is outside this path (and multiplies by exactly that zero in the reference, Bwd.cu:532-553).
        out = dict(v_means2d=torch.zeros(nnz, 2, **f32), v_ray_transforms=torch.zeros(nnz, 3, 3, **f32),
                   v_colors=torch.zeros(nnz, 3, **f32), v_opacities=torch.zeros(nnz, **f32),
                   v_normals=torch.zeros(nnz, 3, **f32), v_densify=torch.zeros(nnz, 2, **f32))
        if want_abs:
            out["v_means2d_abs"] = torch.zeros(nnz, 2, **f32)
        if nnz > 0 and flatten_ids.shape[0] > 0:
            cabi.raster2dgs_bwd(C, width, height, tile_size, 3, nnz, counts, means2d, ray_transforms, colors, opacities,
                                normals, bg if has_bg else None, isect_offsets, flatten_ids, render_alphas, render_Ts,
                                last_ids, median_ids, v_colors, v_depths, v_alphas, v_normals, v_median, out, _ws(dev))
        v_bg = None
        if has_bg and ctx.needs_input_grad[6]:
            v_bg = (v_colors * (1.0 - render_alphas)).sum((1, 2))  # GSC/rasterize_to_pixels.cpp:254-261
        return (out["v_means2d"], out["v_ray_transforms"], out["v_colors"], out["v_opacities"], out["v_normals"],
                out["v_densify"], v_bg, None, None, None, None, None, None, out.get("v_means2d_abs"), None)


def rasterize_to_pixels_2dgs(means2d, ray_transforms, colors, opacities, normals, densify, image_width, image_height,
                             tile_size, isect_offsets, flatten_ids, backgrounds=None, masks=None, packed=False, absgrad=None,
                             distloss=False):
    """-> (render_colors, render_depths, render_alphas, render_normals, render_distort, render_median, visibilities)."""
    C = isect_offsets.shape[0]
    _check(packed, "gssdf_b200 implements the packed layout only")
    nnz = means2d.shape[0]
    _check(tuple(means2d.shape) == (nnz, 2), "Invalid shape for means2d")
    _check(tuple(ray_transforms.shape) == (nnz, 3, 3), "Invalid shape for conics")
    _check(colors.shape[0] == nnz, f"Invalid shape for colors {colors.shape[0]}, {nnz}")
    _check(tuple(opacities.shape) == (nnz,), f"Invalid shape for opacities {tuple(opacities.shape)}, {nnz}")
    channels = colors.shape[-1]
    if channels > 512 or channels == 0:
        raise ValueError(f"Unsupported number of color channels: {channels}")  # std::invalid_argument in the reference
    if backgrounds is not None:
        _check(tuple(backgrounds.shape) == (C, channels), "Invalid shape for backgrounds")
        backgrounds = backgrounds.contiguous()
    _check(masks is None, "tile masks are outside the GS-SDF path (always nullopt, neural_gaussian.cpp:223)")
    th, tw = isect_offsets.shape[1], isect_offsets.shape[2]
    _check(th * tile_size >= image_height, "Assert Failed: tile_height * tile_size >= image_height")
    _check(tw * tile_size >= image_width, "Assert Failed: tile_width * tile_size >= image_width")
    for t in (means2d, ray_transforms, colors, opacities, normals, densify, isect_offsets, flatten_ids):
        _check(t.is_contiguous(), "inputs must be contiguous")
    return RasterizeToPixels2DGS.apply(means2d, ray_transforms, colors, opacities, normals, densify, backgrounds, masks,
                                       image_width, image_height, tile_size, isect_offsets, flatten_ids, absgrad, distloss)


# ----------------------------------------------------------------------------------------------
# the caller: rasterization_2dgs_sdf (neural_gaussian.cpp:129-271), line for line in call order
# ----------------------------------------------------------------------------------------------
def rasterization_2dgs_sdf(means, quats, scales, opacities, colors, viewmats, Ks, width, height, render_mode="RGB+ED",
                           near_plane=0.05, far_plane=300.0, radius_clip=0.0, sh_degree=None, packed=True, tile_size=16,
                           backgrounds=None, sparse_grad=False, absgrad=False, distloss=False, randns=None):
    N, C = means.shape[0], viewmats.shape[0]
    _check(tuple(opacities.shape) == (N,), "Invalid opacities shape")
    _check(render_mode in ("RGB", "D", "ED", "RGB+D", "RGB+ED"), "Invalid render_mode")
    (camera_ids, gaussian_ids, radii, means2d, depths, ray_transforms, normals, samples,
     samples_weights) = fully_fused_projection_2dgs(means, quats, scales, viewmats, Ks, width, height, near_plane, far_plane,
                                                    radius_clip, packed, sparse_grad, randns=randns)
    pt_opacities = opacities[gaussian_ids]
    pt_colors = get_view_colors(viewmats, means, radii, colors, camera_ids, gaussian_ids, sh_degree)
    _tpg, flatten_ids, isect_offsets = tile_encode(width, height, tile_size, means2d, radii, depths, packed, C, camera_ids,
                                                   gaussian_ids)
    means2d_absgrad = torch.zeros_like(means2d).requires_grad_(absgrad)
    densify = torch.zeros_like(means2d).requires_grad_(True)
    (render_colors, render_depths, render_alphas, render_normals, render_distort, render_median,
     visibilities) = rasterize_to_pixels_2dgs(means2d, ray_transforms, pt_colors, pt_opacities, normals, densify, width, height,
                                              tile_size, isect_offsets, flatten_ids, backgrounds, None, packed,
                                              means2d_absgrad, distloss)
    meta = {}
    if absgrad:
        meta["absgrad"] = means2d_absgrad
    if render_mode in ("ED", "RGB+ED"):
        render_depths = (render_depths / render_alphas).nan_to_num()
    render_colors = torch.cat([render_colors, render_depths], -1)
    render_normals = render_normals.matmul(viewmats.inverse()[0, :3, :3].t())
    meta.update(render_normal=render_normals, render_median=render_median, normal=normals, gaussian_ids=gaussian_ids,
                radii=radii, gradient_2dgs=densify, samples=samples, samples_weights=samples_weights,
                samples_opacities=pt_opacities, visibilities=visibilities, render_distort=render_distort,
                flatten_ids=flatten_ids, isect_offsets=isect_offsets, means2d=means2d, depths=depths,
                ray_transforms=ray_transforms, colors=pt_colors, camera_ids=camera_ids)
    return render_colors, render_alphas, meta
