"""TEST INFRASTRUCTURE ONLY. Compiles the reference's simple-knn (submodules/simple-knn/spatial.cu, simple_knn.cu and ext.cpp) from where
they lie under the reference sources (never copied) into oracle/_ref/simple_knn_ref.so for sm_90a, the torch extension `simple_knn_ref`
with the reference's one function distCUDA2. The reference builds the `simple-knn` target (CMakeLists.txt:141-144) under
CMAKE_BUILD_TYPE RelWithDebInfo (`-O2 -g -DNDEBUG`, :6) followed by the directory-wide add_definitions(-O3 -DWITH_CUDA
-DTHRUST_IGNORE_CUB_VERSION_CHECK) (:12), so the last -O3 wins; no fast-math, so its division is IEEE. The same flags are used here.
simple_knn.cu uses FLT_MAX without including <cfloat>, which this toolkit's headers no longer pull in, so `-include cfloat` is passed
on the command line and the source stays untouched. Output stays out of git (oracle/_ref/ is ignored)."""
import os
import subprocess
import sys
import sysconfig

HERE = os.path.dirname(os.path.abspath(__file__))
KNN = "/root/reference/submodules/simple-knn"
OUT_DIR = os.path.join(HERE, "_ref")


def available():
    """True where the reference sources can be read; elsewhere there is nothing to compile."""
    return os.access(os.path.join(KNN, "simple_knn.cu"), os.R_OK)


def build(force=False):
    import torch
    from torch.utils import cpp_extension as ce
    os.makedirs(OUT_DIR, exist_ok=True)
    out = os.path.join(OUT_DIR, "simple_knn_ref.so")
    if os.path.exists(out) and not force:
        return out
    inc = [f"-I{KNN}", f"-I{sysconfig.get_paths()['include']}"] + [f"-I{p}" for p in ce.include_paths("cuda")]
    defs = ["-DTORCH_EXTENSION_NAME=simple_knn_ref", "-DTORCH_API_INCLUDE_EXTENSION_H", "-D_GLIBCXX_USE_CXX11_ABI=1"]
    nvcc = "/usr/local/cuda/bin/nvcc"
    ref_flags = ["-O2", "-g", "-DNDEBUG", "-O3", "-DWITH_CUDA", "-DTHRUST_IGNORE_CUB_VERSION_CHECK"]
    cu = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-Xcompiler", "-fPIC", "-ccbin", "/usr/bin/g++", "-w",
          "-include", "cfloat"] + ref_flags
    jobs = [(cu, os.path.join(KNN, "simple_knn.cu")), (cu, os.path.join(KNN, "spatial.cu")),
            (["/usr/bin/g++", "-std=c++17", "-fPIC", "-w"] + ref_flags, os.path.join(KNN, "ext.cpp"))]
    objs, procs = [], []
    for cmd, src in jobs:
        o = os.path.join(OUT_DIR, "knn_" + os.path.basename(src) + ".o")
        objs.append(o)
        procs.append((src, subprocess.Popen(cmd + inc + defs + ["-c", src, "-o", o], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for name, p in procs:
        log, _ = p.communicate()
        if p.returncode:
            sys.stderr.write(log)
            raise RuntimeError("reference build failed on " + name)
    libdir = os.path.join(os.path.dirname(torch.__file__), "lib")
    subprocess.check_call(["/usr/bin/g++", "-shared", "-o", out + ".tmp"] + objs +
                          [f"-L{libdir}", "-ltorch", "-ltorch_cpu", "-ltorch_cuda", "-lc10", "-lc10_cuda", "-ltorch_python",
                           "-L/usr/local/cuda/lib64", "-lcudart", f"-Wl,-rpath,{libdir}"])
    os.replace(out + ".tmp", out)
    for o in objs:
        os.remove(o)
    return out


if __name__ == "__main__":
    print(build(force="-f" in sys.argv))
