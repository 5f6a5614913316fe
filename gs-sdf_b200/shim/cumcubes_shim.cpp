// cumcubes twin (shim/include/cumcubes.hpp) over the C ABI: mc::marching_cubes -> gssdf_marching_cubes; mc::save_mesh_as_ply writes
// the byte layout of the reference's writer (include/mesher/cumcubes/src/cumcubes.cpp:30-80).
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>

#include <array>
#include <fstream>
#include <stdexcept>

#include "../../include/gssdf_b200.h"
#include "cumcubes.hpp"

namespace {
void check(int rc) {
    static const bool abi_ok = gssdf_abi_revision() == GSSDF_ABI_REVISION;
    TORCH_CHECK(abi_ok, "gssdf_b200 cumcubes shim was compiled against ABI revision ", GSSDF_ABI_REVISION,
                " but libgssdf_b200.so is revision ", gssdf_abi_revision(), ": rebuild the shim");
    if (rc == GSSDF_EINVAL) throw std::invalid_argument(std::string("gssdf_b200: ") + gssdf_last_error());
    if (rc != GSSDF_OK) throw std::runtime_error(std::string("gssdf_b200: ") + gssdf_last_error());
}

// one call with the given capacities; returns {n_vertices, n_faces, overflow}
std::array<int32_t, 3> run(const Tensor &grid, float thresh, const float *lower, const float *upper, Tensor &vertices, Tensor &faces,
                           Tensor &counts, Tensor &ws) {
    gssdf_marching_cubes_args a{};
    a.nx = (int32_t)grid.size(0), a.ny = (int32_t)grid.size(1), a.nz = (int32_t)grid.size(2);
    a.grid = grid.data_ptr<float>();
    a.thresh = thresh;
    for (int k = 0; k < 3; ++k) a.lower[k] = lower[k], a.upper[k] = upper[k];
    a.vertex_cap = vertices.size(0), a.face_cap = faces.size(0);
    a.vertices = vertices.data_ptr<float>();
    a.faces = faces.data_ptr<int32_t>();
    a.counts = counts.data_ptr<int32_t>();
    a.workspace = ws.data_ptr();
    a.workspace_bytes = (size_t)ws.numel();
    check(gssdf_marching_cubes(&a, reinterpret_cast<gssdf_stream_t>(at::cuda::getCurrentCUDAStream().stream())));
    auto h = counts.cpu();  // the reference reads its counts back too (cumcubes_kernel.cu:236-237)
    const int32_t *c = h.data_ptr<int32_t>();
    return {c[0], c[1], c[2]};
}
}  // namespace

std::vector<Tensor> mc::marching_cubes(const Tensor &density_grid, const float thresh, const std::vector<float> lower,
                                       const std::vector<float> upper) {
    CHECK_INPUT(density_grid);
    TORCH_CHECK(density_grid.ndimension() == 3);
    TORCH_CHECK(lower.size() == 3 && upper.size() == 3, "lower and upper need 3 values each");
    return mc::marching_cubes_wrapper(density_grid, thresh, lower.data(), upper.data());
}

std::vector<Tensor> mc::marching_cubes_wrapper(const Tensor &density_grid, const float thresh, const float *lower, const float *upper) {
    CHECK_INPUT(density_grid);
    TORCH_CHECK(density_grid.ndimension() == 3 && density_grid.scalar_type() == torch::kFloat, "density_grid must be float32 [nx,ny,nz]");
    const c10::cuda::CUDAGuard guard(density_grid.device());
    const auto opt = density_grid.options();
    const int64_t n = density_grid.numel();
    Tensor ws = torch::empty({(int64_t)std::max<size_t>(
                                 gssdf_marching_cubes_workspace_bytes((int32_t)density_grid.size(0), (int32_t)density_grid.size(1),
                                                                      (int32_t)density_grid.size(2)), 1)},
                             opt.dtype(torch::kUInt8));
    Tensor counts = torch::zeros({4}, opt.dtype(torch::kInt));
    // first guess at the sizes; on overflow the call is repeated once with the exact counts it reported
    int64_t vcap = std::max<int64_t>(n / 16, 1024), fcap = 2 * vcap;
    for (int attempt = 0; attempt < 2; ++attempt) {
        Tensor vertices = torch::empty({vcap, 3}, opt);
        Tensor faces = torch::empty({fcap, 3}, opt.dtype(torch::kInt));
        auto c = run(density_grid, thresh, lower, upper, vertices, faces, counts, ws);
        if (!c[2]) return {vertices.slice(0, 0, c[0]), faces.slice(0, 0, c[1])};
        vcap = std::max<int64_t>(c[0], 1), fcap = std::max<int64_t>(c[1], 1);
    }
    throw std::runtime_error("gssdf_b200: marching_cubes overflowed its exact capacities");
}

void mc::save_mesh_as_ply(const std::string filename, Tensor vertices, Tensor faces, Tensor colors) {
    CHECK_CONTIGUOUS(vertices);
    CHECK_CONTIGUOUS(faces);
    CHECK_CONTIGUOUS(colors);
    TORCH_CHECK(colors.scalar_type() == torch::kUInt8, "colors must be uint8");
    TORCH_CHECK(vertices.scalar_type() == torch::kFloat && faces.scalar_type() == torch::kInt, "vertices float32, faces int32");
    TORCH_CHECK(colors.size(0) == vertices.size(0), "one colour per vertex");
    vertices = vertices.cpu().contiguous();
    faces = faces.cpu().contiguous();
    colors = colors.cpu().contiguous();
    std::ofstream f(filename, std::ios::out | std::ios::binary);
    TORCH_CHECK(f.good(), "cannot open ", filename);
    f << "ply\nformat binary_little_endian 1.0\nelement vertex " << vertices.size(0) << "\n"
      << "property float x\nproperty float y\nproperty float z\nproperty uchar red\nproperty uchar green\nproperty uchar blue\n"
      << "element face " << faces.size(0) << "\nproperty list int int vertex_index\nend_header\n";
    const float *v = vertices.data_ptr<float>();
    const uint8_t *c = colors.data_ptr<uint8_t>();
    for (int64_t i = 0; i < vertices.size(0); ++i) {
        f.write(reinterpret_cast<const char *>(v + 3 * i), 3 * sizeof(float));
        f.write(reinterpret_cast<const char *>(c + 3 * i), 3);
    }
    const int32_t *fc = faces.data_ptr<int32_t>();
    const int32_t three = 3;
    for (int64_t i = 0; i < faces.size(0); ++i) {
        f.write(reinterpret_cast<const char *>(&three), sizeof(int32_t));
        f.write(reinterpret_cast<const char *>(fc + 3 * i), 3 * sizeof(int32_t));
    }
}
