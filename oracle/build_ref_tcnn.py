"""TEST INFRASTRUCTURE ONLY. Compiles oracle/ref_tcnn_grid_driver.cu against tiny-cuda-nn's HEADERS where they lie under /root/reference
(header-only use of encodings/grid.h; tcnn's own build system, its .cu translation units and its runtime are not used) into
oracle/_ref/tcnn_grid_ref.so for sm_90a. Output stays out of git (oracle/_ref/ is ignored)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
TCNN = "/root/reference/submodules/tcnn_binding/submodules/tiny-cuda-nn"
OUT = os.path.join(HERE, "_ref", "tcnn_grid_ref.so")


def available():
    """True where tiny-cuda-nn's headers can be read (the build container); elsewhere there is nothing to compile."""
    return os.access(os.path.join(TCNN, "include"), os.R_OK | os.X_OK)


def build(force=False):
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    if os.path.exists(OUT) and not force:
        return OUT
    if not os.path.isdir(TCNN):
        raise RuntimeError("/root/reference is not present: the tcnn reference kernels can only be built in the build container")
    cmd = ["/usr/local/cuda/bin/nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--extended-lambda",
           "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC", "-ccbin", "/usr/bin/g++", "-w", "-DTCNN_MIN_GPU_ARCH=90",
           f"-I{TCNN}/include", f"-I{TCNN}/dependencies", f"-I{TCNN}/dependencies/fmt/include", f"-I{TCNN}/dependencies/cutlass/include",
           "-DFMT_HEADER_ONLY", "-shared", os.path.join(HERE, "ref_tcnn_grid_driver.cu"), "-o", OUT, "-lcudart"]
    p = subprocess.run(cmd, capture_output=True, text=True)
    if p.returncode:
        sys.stderr.write(p.stdout + p.stderr)
        raise RuntimeError("tcnn reference driver failed to build")
    return OUT


if __name__ == "__main__":
    print(build(force="-f" in sys.argv))
