// Twin of the reference's include/mesher/cumcubes/include/cumcubes.hpp: same namespace, names and signatures, so that
// include/neural_net/local_map.cpp (LocalMap::meshing_) and include/mesher/mesher.cpp compile and link unchanged against
// gs-sdf_b200/shim/cumcubes_shim.cpp, which runs gssdf_marching_cubes (include/gssdf_b200.h) instead of the cumcubes kernels.
#pragma once
#include <cuda_runtime.h>
#include <torch/torch.h>

using torch::Tensor;

namespace mc {
// {vertices [V,3] float32, faces [F,3] int32} on the grid's device; vertices in lattice-edge order, faces in cell order
std::vector<Tensor> marching_cubes(const Tensor &, const float, const std::vector<float>, const std::vector<float>);
std::vector<Tensor> marching_cubes_wrapper(const Tensor &, const float, const float *, const float *);
// binary PLY: float x y z + uchar red green blue per vertex, `list int int vertex_index` per face
void save_mesh_as_ply(const std::string, Tensor, Tensor, Tensor);
}  // namespace mc

#define CHECK_CUDA(x) TORCH_CHECK(x.is_cuda(), #x " must be a CUDA tensor")
#define CHECK_CPU(x) TORCH_CHECK(!x.is_cuda(), #x " must be a CPU tensor")
#define CHECK_CONTIGUOUS(x) TORCH_CHECK(x.is_contiguous(), #x " must be contiguous")
#define CHECK_INPUT(x) \
    CHECK_CUDA(x);     \
    CHECK_CONTIGUOUS(x)
#define CHECK_CPU_INPUT(x) \
    CHECK_CPU(x);          \
    CHECK_CONTIGUOUS(x)
