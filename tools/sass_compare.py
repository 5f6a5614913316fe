"""Compare the SASS of kernels across a source change: a kernel that became a template must compile, in its plain instantiation, to the
instructions the untemplated kernel compiled to (symbol names aside).

    python tools/sass_compare.py [--rev HEAD~1]

compiles gs-sdf_b200/csrc/{raster,loss}.cu of the working tree and of `rev` (with that revision's headers) for sm_90a with build.py's
flags, disassembles both with cuobjdump -sass and compares the instruction streams of the kernel pairs in PAIRS (addresses and
encodings dropped). Needs nvcc and cuobjdump, no GPU. Exit code 1 if a pair differs or is missing."""
import argparse
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "gs-sdf_b200"))
from build import NVCC_FLAGS  # noqa: E402

CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")
# (source, kernel symbol before, plain instantiation after)
PAIRS = [
    ("raster.cu", "_ZN5gssdf22render_post_fwd_kernelE26gssdf_render_post_fwd_args",
     "_ZN5gssdf22render_post_fwd_kernelILi0EEEv26gssdf_render_post_fwd_argsPKf"),
    ("raster.cu", "_ZN5gssdf22render_post_bwd_kernelE26gssdf_render_post_bwd_args",
     "_ZN5gssdf22render_post_bwd_kernelILi0EEEv26gssdf_render_post_bwd_argsPKf"),
    ("raster.cu", "_ZN5gssdf14l1_loss_kernelE18gssdf_l1_loss_argsl", "_ZN5gssdf14l1_loss_kernelILb0EEEv18gssdf_l1_loss_argslPKh"),
    ("loss.cu", "_ZN5gssdf16dssim_fwd_kernelE21gssdf_dssim_loss_argsNS_10SsimWindowEPfNS_7SsimSumEi",
     "_ZN5gssdf16dssim_fwd_kernelILb0EEEv21gssdf_dssim_loss_argsNS_10SsimWindowEPfNS_7SsimSumEiPKh"),
    ("loss.cu", "_ZN5gssdf16dssim_bwd_kernelE21gssdf_dssim_loss_argsNS_10SsimWindowEPKffi",
     "_ZN5gssdf16dssim_bwd_kernelILb0EEEv21gssdf_dssim_loss_argsNS_10SsimWindowEPKffiPKh"),
]


def _compile(src, obj):
    cmd = [os.path.join(CUDA, "bin", "nvcc")] + [f for f in NVCC_FLAGS if f not in ("-Xptxas", "-v")] + ["-c", src, "-o", obj]
    subprocess.run(cmd, check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)


def sass_functions(obj):
    """{symbol: [instruction text]} of every kernel in the object."""
    out = subprocess.run([os.path.join(CUDA, "bin", "cuobjdump"), "-sass", obj], check=True, capture_output=True, text=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = funcs.setdefault(m.group(1), [])
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s*(.*?)\s*;?\s*/\*", line)
        if cur is not None and m:
            cur.append(m.group(1).rstrip(" ;"))
    return funcs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rev", default="HEAD", help="git revision to compare the working tree against")
    args = ap.parse_args()
    ok = True
    with tempfile.TemporaryDirectory() as tmp:
        old = os.path.join(tmp, "old")
        os.makedirs(old)
        # the revision's csrc/ and include/ in their repository layout (the sources include ../../include/gssdf_b200.h)
        arc = subprocess.run(["git", "-C", ROOT, "archive", args.rev, "gs-sdf_b200/csrc", "include"], check=True, capture_output=True).stdout
        subprocess.run(["tar", "-x", "-C", old], input=arc, check=True)
        objs = {}
        for src in sorted({p[0] for p in PAIRS}):
            for tag, base in (("old", old), ("new", ROOT)):
                o = os.path.join(tmp, f"{tag}_{src}.o")
                _compile(os.path.join(base, "gs-sdf_b200", "csrc", src), o)
                objs[tag, src] = sass_functions(o)
        for src, before, after in PAIRS:
            a, b = objs["old", src].get(before), objs["new", src].get(after)
            if a is None or b is None:
                print(f"MISSING {src}: {before if a is None else after}")
                ok = False
                continue
            same = a == b
            ok &= same
            print(f"{'same' if same else 'DIFFERENT':9s} {len(a):5d} vs {len(b):5d} instructions  {src}: {after}")
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
