// libtorch twin of simple-knn's spatial.h (submodules/simple-knn): the one function neural_gaussian.cpp calls, declared in the global
// namespace as simple-knn declares it, so that `#include "spatial.h"` resolves here and neural_gaussian.cpp compiles unchanged
// (INTEGRATION 3h). Implemented in shim/simple_knn_shim.cpp over gssdf_knn3_mean_dist2 (include/gssdf_b200.h f-10; DESIGN 7k).
#pragma once
#include <torch/torch.h>

// points: CUDA float32 [P,3] (made contiguous). Returns float32 [P] on the points' device: for each point the mean of its three
// smallest squared distances to the other points, bit-identical to simple-knn's distCUDA2.
torch::Tensor distCUDA2(const torch::Tensor &points);
