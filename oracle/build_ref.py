"""TEST INFRASTRUCTURE ONLY. Compiles the reference fork's 2DGS CUDA kernels from where they lie under
the reference sources (never copied) + oracle/ref_driver.cpp into oracle/_ref/gsplat_ref.so for sm_90a, with
the reference's own flags (submodules/gsplat_cpp/CMakeLists.txt:13-17: -O3 --use_fast_math
--expt-relaxed-constexpr). Only the five kernel translation units on the GS-SDF path are built; the
reference's cmake build system is not run. Output stays out of git (oracle/_ref/ is ignored)."""
import os
import subprocess
import sys
import sysconfig

HERE = os.path.dirname(os.path.abspath(__file__))
GSF = "/root/reference/submodules/gsplat_cpp/submodules/gsplat/gsplat/cuda"
OUT_DIR = os.path.join(HERE, "_ref")
KERNELS = ["Projection2DGSPacked.cu", "IntersectTile.cu", "RasterizeToPixels2DGSFwd.cu", "RasterizeToPixels2DGSBwd.cu",
           "SphericalHarmonicsCUDA.cu"]


def available():
    """True where the reference sources can be read (the build container); elsewhere there is nothing to compile."""
    return os.access(os.path.join(GSF, "csrc"), os.R_OK | os.X_OK)


def build(force=False):
    import torch
    from torch.utils import cpp_extension as ce
    os.makedirs(OUT_DIR, exist_ok=True)
    out = os.path.join(OUT_DIR, "gsplat_ref.so")
    if os.path.exists(out) and not force:
        return out
    if not os.path.isdir(GSF):
        raise RuntimeError("/root/reference is not present: the reference oracle can only be built in the build container")
    inc = [f"-I{GSF}/include", f"-I{GSF}/csrc", f"-I{GSF}/csrc/third_party/glm", f"-I{sysconfig.get_paths()['include']}"]
    inc += [f"-I{p}" for p in ce.include_paths("cuda")]
    defs = ["-DTORCH_EXTENSION_NAME=gsplat_ref", "-DTORCH_API_INCLUDE_EXTENSION_H", "-D_GLIBCXX_USE_CXX11_ABI=1",
            "-DGLM_FORCE_CUDA", "-DGLM_ENABLE_EXPERIMENTAL"]
    nvcc = "/usr/local/cuda/bin/nvcc"
    common = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "--use_fast_math", "--expt-relaxed-constexpr", "-std=c++17",
              "-Xcompiler", "-fPIC", "-ccbin", "/usr/bin/g++", "-w"]
    objs, procs = [], []
    for k in KERNELS:
        o = os.path.join(OUT_DIR, k + ".o")
        objs.append(o)
        procs.append((k, subprocess.Popen([nvcc] + common + inc + defs + ["-c", os.path.join(GSF, "csrc", k), "-o", o],
                                          stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    o = os.path.join(OUT_DIR, "ref_driver.o")
    objs.append(o)
    procs.append(("ref_driver.cpp", subprocess.Popen(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-w"] + inc + defs +
                                                     ["-c", os.path.join(HERE, "ref_driver.cpp"), "-o", o],
                                                     stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for name, p in procs:
        log, _ = p.communicate()
        if p.returncode:
            sys.stderr.write(log)
            raise RuntimeError("reference build failed on " + name)
    libdir = os.path.join(os.path.dirname(torch.__file__), "lib")
    subprocess.check_call(["/usr/bin/g++", "-shared", "-o", out] + objs +
                          [f"-L{libdir}", "-ltorch", "-ltorch_cpu", "-ltorch_cuda", "-lc10", "-lc10_cuda", "-ltorch_python",
                           "-L/usr/local/cuda/lib64", "-lcudart", f"-Wl,-rpath,{libdir}"])
    for o in objs:
        os.remove(o)
    return out


if __name__ == "__main__":
    print(build(force="-f" in sys.argv))
