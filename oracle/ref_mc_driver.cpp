// TEST INFRASTRUCTURE ONLY. pybind11 module around the reference's UNMODIFIED mc::marching_cubes (include/mesher/cumcubes/src/
// cumcubes.cpp + cumcubes_kernel.cu, compiled from where they lie by oracle/build_ref_mc.py into oracle/_ref/cumcubes_ref.so). It lets
// the GPU tests and oracle/gen_golden_mc.py run the reference's marching-cubes kernels on the same fields as ours.
#include <torch/extension.h>

#include "cumcubes.hpp"

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) { m.def("marching_cubes", &mc::marching_cubes); }
