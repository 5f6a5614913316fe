"""Builds libgssdf_b200.so (hand-written sm_90a CUDA behind the C ABI of include/gssdf_b200.h)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libgssdf_b200.so")
SOURCES = ["api.cu", "project.cu", "sh.cu", "tiles.cu", "raster.cu", "sdf.cu", "sdf_tc.cu", "loss.cu", "grid_ops.cu", "optim.cu", "octree.cu", "densify.cu", "mesh.cu", "sdf_mesh.cu", "gs_init.cu", "mesh_cull.cu", "octree_build.cu", "mesh_eval.cu", "knn.cu", "image_metrics.cu", "outlier.cu", "nsdf.cu", "frames.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
              "--extended-lambda", "-Xcompiler", "-fPIC", "-Xptxas", "-v"]


def build(verbose=False, force=False):
    srcs = [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    deps = srcs + [os.path.join(CSRC, "common.cuh"), os.path.join(CSRC, "adam.cuh"), os.path.join(CSRC, "sdf_grid.cuh"), os.path.join(CSRC, "conic.cuh"), os.path.join(CSRC, "sdf_loss.cuh"), os.path.join(CSRC, "mc_table.h"), os.path.join(CSRC, "octree_query.cuh"), os.path.join(CSRC, "morton.cuh"), os.path.join(CSRC, "depth_normal.cuh"), os.path.join(HERE, "..", "include", "gssdf_b200.h")]
    if not force and os.path.exists(OUT) and all(os.path.getmtime(d) <= os.path.getmtime(OUT) for d in deps):
        return OUT
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for s in srcs:
        o = os.path.join(HERE, "build", os.path.basename(s) + ".o")
        objs.append(o)
        if not force and os.path.exists(o) and all(os.path.getmtime(d) <= os.path.getmtime(o) for d in [s] + deps[len(srcs):]):
            continue
        cmd = [nvcc] + NVCC_FLAGS + ["-ccbin", "/usr/bin/g++", "-c", s, "-o", o]
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for s, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode:
            sys.stderr.write(out)
        if p.returncode:
            raise RuntimeError("nvcc failed on " + s)
    # link next to the target and rename: a concurrent reader never sees a half-written library
    subprocess.check_call([nvcc, "-shared", "-o", OUT + ".tmp"] + objs + ["-ccbin", "/usr/bin/g++", "-lcudart"])
    os.replace(OUT + ".tmp", OUT)
    return OUT


SHIM_OUT = os.path.join(HERE, "gssdf_shim.so")


def build_shim(force=False):
    """libtorch shim (gs-sdf_b200/shim/) + its pybind harness -> gssdf_shim.so, linked against libgssdf_b200.so."""
    import sysconfig

    import torch
    srcs = [os.path.join(HERE, "shim", f) for f in ("gsplat_cpp_shim.cpp", "tcnn_binding_shim.cpp", "cumcubes_shim.cpp", "gssdf_mesh.cpp", "gssdf_metrics.cpp", "gssdf_init.cpp", "gssdf_octree.cpp", "gssdf_outlier.cpp", "gssdf_frames.cpp", "simple_knn_shim.cpp", "py_binding.cpp")]
    deps = srcs + [os.path.join(HERE, "shim", "include", "gsplat_cpp", h) for h in ("fully_fused_projection.h", "rasterize_to_pixels.h", "rendering.h")]
    deps.append(os.path.join(HERE, "shim", "include", "tcnn_binding", "tcnn_binding.h"))
    deps.append(os.path.join(HERE, "shim", "include", "cumcubes.hpp"))
    deps += [os.path.join(HERE, "shim", "include", h) for h in ("gssdf_mesh.hpp", "gssdf_metrics.hpp", "gssdf_frames.hpp", "gssdf_init.hpp", "gssdf_sdf_net.hpp", "gssdf_octree.hpp", "spatial.h")]
    deps.append(os.path.join(HERE, "..", "include", "gssdf_b200.h"))
    if not force and os.path.exists(SHIM_OUT) and all(os.path.getmtime(d) <= os.path.getmtime(SHIM_OUT) for d in deps):
        return SHIM_OUT
    tdir = os.path.dirname(torch.__file__)
    inc = [f"-I{os.path.join(HERE, 'shim', 'include')}", f"-I{tdir}/include", f"-I{tdir}/include/torch/csrc/api/include",
           "-I/usr/local/cuda/include", f"-I{sysconfig.get_paths()['include']}"]
    # nlohmann::json for the tcnn_binding twin: the reference gets it from tiny-cuda-nn/dependencies (json/json.hpp); this image carries
    # the same single header under cudnn_frontend's third-party directory
    import glob
    js = glob.glob(os.path.join(sysconfig.get_paths()["purelib"], "include", "cudnn_frontend", "thirdparty"))
    inc += [f"-I{p_}" for p_ in js]
    flags = ["-std=c++17", "-O2", "-fPIC", "-w", "-D_GLIBCXX_USE_CXX11_ABI=1", "-DTORCH_EXTENSION_NAME=gssdf_shim", "-DTORCH_API_INCLUDE_EXTENSION_H"]
    objs, procs = [], []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for s_ in srcs:
        o = os.path.join(HERE, "build", os.path.basename(s_) + ".o")
        objs.append(o)
        procs.append((s_, subprocess.Popen(["/usr/bin/g++"] + flags + inc + ["-c", s_, "-o", o], stdout=subprocess.PIPE,
                                           stderr=subprocess.STDOUT, text=True)))
    for s_, p in procs:
        out, _ = p.communicate()
        if p.returncode:
            sys.stderr.write(out)
            raise RuntimeError("g++ failed on " + s_)
    subprocess.check_call(["/usr/bin/g++", "-shared", "-o", SHIM_OUT + ".tmp"] + objs +
                          [f"-L{HERE}", "-l:libgssdf_b200.so", f"-L{tdir}/lib", "-ltorch", "-ltorch_cpu", "-ltorch_cuda", "-lc10", "-lc10_cuda",
                           "-ltorch_python", "-L/usr/local/cuda/lib64", "-lcudart", f"-Wl,-rpath,{tdir}/lib", "-Wl,-rpath,$ORIGIN"])
    os.replace(SHIM_OUT + ".tmp", SHIM_OUT)
    return SHIM_OUT


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv, force="-f" in sys.argv))
    if "--no-shim" not in sys.argv:  # the shim embeds the argument-struct layouts: always keep it in step with the header
        print(build_shim(force="-f" in sys.argv))
