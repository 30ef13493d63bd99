"""Builds libfbgpu.so (CUDA, sm_90a: H100) and libfbdatagen.so in-tree."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = "arch=compute_90a,code=sm_90a"      # H100 (Hopper)


def _stale(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources if os.path.exists(s))


def build_fbgpu(force=False, verbose=False, defines=None, out_name="libfbgpu.so"):
    src = os.path.join(HERE, "csrc", "fbgpu.cu")
    deps = [src, os.path.join(HERE, "csrc", "kernels.cuh"), os.path.join(HERE, "csrc", "fbgpu_types.h"), os.path.join(HERE, "csrc", "stripe.h"), os.path.join(HERE, "csrc", "rbf_reader.h"), os.path.join(HERE, "csrc", "bitaddr.h"), os.path.join(HERE, "csrc", "program_compiler.h"), os.path.join(HERE, "csrc", "roaring_parse.h"), os.path.join(HERE, "csrc", "host_error.h"), os.path.join(HERE, "csrc", "wp_machine.h"), os.path.join(HERE, "csrc", "resolve.h"), os.path.join(HERE, "csrc", "node.h"),
            os.path.join(ROOT, "include", "fbgpu.h")]
    out = os.path.join(HERE, out_name)
    if force or _stale(out, deps):
        cmd = [NVCC, "-O3", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-lineinfo",
               "-gencode", ARCH, "-o", out, src, "-ldl"]
        for d in (defines or []):
            cmd.insert(1, "-D" + d)
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        subprocess.check_call(cmd)
    return out


def build_datagen(force=False):
    src = os.path.join(ROOT, "tools", "fbdatagen.c")
    out = os.path.join(ROOT, "tools", "libfbdatagen.so")
    if force or _stale(out, [src]):
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-shared", "-std=gnu11", "-o", out, src, "-lm", "-lpthread"])
    return out


if __name__ == "__main__":
    build_fbgpu(force="--force" in sys.argv, verbose="-v" in sys.argv)
    build_datagen(force="--force" in sys.argv)
    print("built")
