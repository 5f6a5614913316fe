// TEST INFRASTRUCTURE ONLY. Thin pybind11 driver around the UNMODIFIED kernel launchers of the reference's
// gsplat fork, compiled from where they lie under /root/reference by oracle/build_ref.py into
// oracle/_ref/gsplat_ref*.so. It exists to run the reference CUDA kernels on a GPU and dump golden
// vectors (oracle/gen_golden_ref.py). The host glue below (two-pass compaction, cumsum, output
// allocation) is written against the launcher declarations in GSF/csrc/{Projection,Intersect,
// Rasterization,SphericalHarmonics}.h and follows the call order of GSF/csrc/Projection.cpp:654-774,
// Intersect.cpp:15-145, Rasterization.cpp:324-612 -- with ONE deliberate difference: `randns` is an
// argument (the reference draws at::randn after its sync) so that goldens are reproducible.
#include <torch/extension.h>

#include <cmath>
#include <tuple>
#include <vector>

#include "Common.h"
#include "Intersect.h"
#include "Projection.h"
#include "Rasterization.h"
#include "SphericalHarmonics.h"

using at::Tensor;

std::vector<Tensor> ref_projection_2dgs_packed_fwd(Tensor means, Tensor quats, Tensor scales, Tensor viewmats, Tensor Ks,
                                                   int64_t W, int64_t H, double near_plane, double far_plane, double radius_clip,
                                                   Tensor randns_cap) {
    uint32_t N = means.size(0), C = viewmats.size(0);
    auto opt = means.options();
    uint32_t bpr = (N + N_THREADS_PACKED - 1) / N_THREADS_PACKED;
    Tensor block_cnts = at::empty({(int64_t)C * bpr}, opt.dtype(at::kInt));
    gsplat::launch_projection_2dgs_packed_fwd_kernel(means, quats, scales, viewmats, Ks, W, H, near_plane, far_plane, radius_clip,
                                                     c10::nullopt, block_cnts, c10::nullopt, c10::nullopt, c10::nullopt, c10::nullopt,
                                                     c10::nullopt, c10::nullopt, c10::nullopt, c10::nullopt, c10::nullopt,
                                                     c10::nullopt);
    Tensor block_accum = at::cumsum(block_cnts, 0, at::kInt);
    int32_t nnz = block_accum[-1].item<int32_t>();
    Tensor indptr = at::empty({C + 1}, opt.dtype(at::kInt));
    Tensor camera_ids = at::empty({nnz}, opt.dtype(at::kLong)), gaussian_ids = at::empty({nnz}, opt.dtype(at::kLong));
    Tensor radii = at::empty({nnz, 2}, opt.dtype(at::kInt)), means2d = at::empty({nnz, 2}, opt), depths = at::empty({nnz}, opt);
    Tensor ray_transforms = at::empty({nnz, 3, 3}, opt), normals = at::empty({nnz, 3}, opt);
    Tensor randns = randns_cap.slice(0, 0, nnz).contiguous();
    Tensor samples = at::empty({nnz, 3}, opt);
    if (nnz)
        gsplat::launch_projection_2dgs_packed_fwd_kernel(means, quats, scales, viewmats, Ks, W, H, near_plane, far_plane,
                                                         radius_clip, block_accum, c10::nullopt, indptr, camera_ids, gaussian_ids,
                                                         radii, means2d, depths, ray_transforms, normals, randns, samples);
    else
        indptr.fill_(0);
    return {indptr, camera_ids, gaussian_ids, radii, means2d, depths, ray_transforms, normals, randns, samples};
}

std::vector<Tensor> ref_projection_2dgs_packed_bwd(Tensor means, Tensor quats, Tensor scales, Tensor viewmats, Tensor Ks, int64_t W,
                                                   int64_t H, Tensor camera_ids, Tensor gaussian_ids, Tensor ray_transforms,
                                                   Tensor randns, Tensor v_means2d, Tensor v_depths, Tensor v_ray_transforms,
                                                   Tensor v_normals, Tensor v_samples) {
    Tensor v_means = at::zeros_like(means), v_quats = at::zeros_like(quats), v_scales = at::zeros_like(scales);
    gsplat::launch_projection_2dgs_packed_bwd_kernel(means, quats, scales, viewmats, Ks, W, H, camera_ids, gaussian_ids,
                                                     ray_transforms, randns, v_means2d, v_depths, v_ray_transforms, v_normals,
                                                     v_samples, false, v_means, v_quats, v_scales, c10::nullopt);
    return {v_means, v_quats, v_scales};
}

Tensor ref_sh_fwd(int64_t degree, Tensor dirs, Tensor coeffs) {
    Tensor colors = at::empty_like(dirs);
    gsplat::launch_spherical_harmonics_fwd_kernel(degree, dirs, coeffs, c10::nullopt, colors);
    return colors;
}

std::vector<Tensor> ref_sh_bwd(int64_t degree, Tensor dirs, Tensor coeffs, Tensor v_colors) {
    Tensor v_coeffs = at::zeros_like(coeffs), v_dirs = at::zeros_like(dirs);
    gsplat::launch_spherical_harmonics_bwd_kernel(degree, dirs, coeffs, c10::nullopt, v_colors, v_coeffs, v_dirs);
    return {v_coeffs, v_dirs};
}

std::vector<Tensor> ref_tile_encode(Tensor means2d, Tensor radii, Tensor depths, Tensor camera_ids, Tensor gaussian_ids, int64_t C,
                                    int64_t tile_size, int64_t tile_width, int64_t tile_height) {
    auto opt = means2d.options();
    int64_t nnz = means2d.size(0);
    uint32_t n_tiles = tile_width * tile_height;
    uint32_t tile_n_bits = (uint32_t)floor(log2(n_tiles)) + 1, cam_n_bits = (uint32_t)floor(log2(C)) + 1;
    Tensor tiles_per_gauss = at::empty({nnz}, opt.dtype(at::kInt));
    int64_t n_isects = 0;
    Tensor cum;
    if (nnz) {
        gsplat::launch_intersect_tile_kernel(means2d, radii, depths, camera_ids, gaussian_ids, C, tile_size, tile_width, tile_height,
                                             c10::nullopt, tiles_per_gauss, c10::nullopt, c10::nullopt);
        cum = at::cumsum(tiles_per_gauss.view({-1}), 0);
        n_isects = cum[-1].item<int64_t>();
    }
    Tensor isect_ids = at::empty({n_isects}, opt.dtype(at::kLong)), flatten_ids = at::empty({n_isects}, opt.dtype(at::kInt));
    if (n_isects)
        gsplat::launch_intersect_tile_kernel(means2d, radii, depths, camera_ids, gaussian_ids, C, tile_size, tile_width, tile_height,
                                             cum, c10::nullopt, isect_ids, flatten_ids);
    Tensor ids_sorted = at::empty_like(isect_ids), flat_sorted = at::empty_like(flatten_ids);
    gsplat::radix_sort_double_buffer(n_isects, tile_n_bits, cam_n_bits, isect_ids, flatten_ids, ids_sorted, flat_sorted);
    Tensor offsets = at::empty({C, tile_height, tile_width}, opt.dtype(at::kInt));
    if (n_isects)
        gsplat::launch_intersect_offset_kernel(ids_sorted, C, tile_width, tile_height, offsets);
    else
        offsets.fill_(0);
    return {tiles_per_gauss, ids_sorted, flat_sorted, offsets};
}

std::vector<Tensor> ref_raster_fwd(Tensor means2d, Tensor ray_transforms, Tensor colors, Tensor opacities, Tensor normals, int64_t W,
                                   int64_t H, int64_t tile_size, Tensor offsets, Tensor flatten_ids) {
    auto opt = means2d.options();
    int64_t C = offsets.size(0), nnz = means2d.size(0);
    Tensor renders = at::empty({C, H, W, 3}, opt), depths = at::empty({C, H, W, 1}, opt), alphas = at::empty({C, H, W, 1}, opt);
    Tensor Ts = at::zeros({C, H, W, 2}, opt), rn = at::empty({C, H, W, 3}, opt), distort = at::empty({C, H, W, 1}, opt);
    Tensor median = at::empty({C, H, W, 1}, opt), last_ids = at::empty({C, H, W}, opt.dtype(at::kInt));
    Tensor median_ids = at::empty({C, H, W}, opt.dtype(at::kInt)), vis = at::zeros({nnz, 1}, opt);
    gsplat::launch_rasterize_to_pixels_2dgs_fwd_kernel<3>(means2d, ray_transforms, colors, opacities, normals, c10::nullopt,
                                                          c10::nullopt, W, H, tile_size, offsets, flatten_ids, renders, depths, alphas,
                                                          Ts, rn, distort, median, last_ids, median_ids, vis);
    return {renders, depths, alphas, Ts, rn, distort, median, last_ids, median_ids, vis};
}

std::vector<Tensor> ref_raster_bwd(Tensor means2d, Tensor ray_transforms, Tensor colors, Tensor opacities, Tensor normals, int64_t W,
                                   int64_t H, int64_t tile_size, Tensor offsets, Tensor flatten_ids, Tensor render_colors,
                                   Tensor render_depths, Tensor render_alphas, Tensor render_Ts, Tensor last_ids, Tensor median_ids,
                                   Tensor v_colors_img, Tensor v_depths_img, Tensor v_alphas_img, Tensor v_normals_img,
                                   Tensor v_distort_img, Tensor v_median_img) {
    Tensor densify = at::zeros_like(means2d);
    Tensor v_means2d = at::zeros_like(means2d), v_rt = at::zeros_like(ray_transforms), v_colors = at::zeros_like(colors);
    Tensor v_opac = at::zeros_like(opacities), v_normals = at::zeros_like(normals), v_densify = at::zeros_like(densify);
    gsplat::launch_rasterize_to_pixels_2dgs_bwd_kernel<3>(means2d, ray_transforms, colors, opacities, normals, densify, c10::nullopt,
                                                          c10::nullopt, W, H, tile_size, offsets, flatten_ids, render_colors,
                                                          render_depths, render_alphas, render_Ts, last_ids, median_ids, v_colors_img,
                                                          v_depths_img, v_alphas_img, v_normals_img, v_distort_img, v_median_img,
                                                          c10::nullopt, v_means2d, v_rt, v_colors, v_opac, v_normals, v_densify);
    return {v_means2d, v_rt, v_colors, v_opac, v_normals, v_densify};
}

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
    m.def("projection_2dgs_packed_fwd", &ref_projection_2dgs_packed_fwd);
    m.def("projection_2dgs_packed_bwd", &ref_projection_2dgs_packed_bwd);
    m.def("sh_fwd", &ref_sh_fwd);
    m.def("sh_bwd", &ref_sh_bwd);
    m.def("tile_encode", &ref_tile_encode);
    m.def("raster_fwd", &ref_raster_fwd);
    m.def("raster_bwd", &ref_raster_bwd);
}
