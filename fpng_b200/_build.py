"""Builds fpng_b200/libfpng_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU)."""
from __future__ import annotations

import glob
import os
import subprocess

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "libfpng_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC,-fvisibility=hidden,-O3", "-shared",
]
# comm.cu binds NCCL at run time (dlopen: the process's own copy if it has one, else the system libnccl.so.2); nothing is linked
LINK_FLAGS = ["-ldl"]


def sources() -> list[str]:
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cpp")))


def is_stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(CSRC, "*.h")) + \
        glob.glob(os.path.join(PKG, "..", "include", "*.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not is_stale():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        nvcc = "nvcc"
    # one object per source, compiled in parallel and only when the source or a header changed; then one link
    from concurrent.futures import ThreadPoolExecutor
    objdir = os.path.join(CSRC, "_obj")
    os.makedirs(objdir, exist_ok=True)
    headers = glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(CSRC, "*.h")) + glob.glob(os.path.join(PKG, "..", "include", "*.h"))
    hdr_time = max(os.path.getmtime(h) for h in headers)
    cflags = [f for f in NVCC_FLAGS if f != "-shared"] + os.environ.get("FPNGB_NVCC_DEFS", "").split()   # e.g. "-DFPNGB_FUSED_TICKET=1" for A/B builds

    def compile_one(src):
        obj = os.path.join(objdir, os.path.basename(src) + ".o")
        if force or not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(src), hdr_time):
            subprocess.check_call([nvcc] + cflags + (["-Xptxas", "-v"] if verbose else []) + ["-c", "-o", obj, src], cwd=CSRC)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        objs = list(ex.map(compile_one, sources()))
    tmp = LIB + ".building"           # not *.so: a half-written library must never be picked up (or shipped to the GPU box)
    subprocess.check_call([nvcc] + NVCC_FLAGS + ["-o", tmp] + objs + LINK_FLAGS, cwd=CSRC)
    os.replace(tmp, LIB)
    return LIB


def build_variant(name: str, defs: str) -> str:
    """Developer A/B builds: the same sources with extra -D macros, into fpng_b200/_variants/libfpng_b200_<name>.so
    (loaded instead of the product library when FPNGB_LIB_VARIANT=<name>; never built or used by default)."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    from concurrent.futures import ThreadPoolExecutor
    objdir = os.path.join(CSRC, "_obj_" + name)
    vdir = os.path.join(PKG, "_variants")
    os.makedirs(objdir, exist_ok=True)
    os.makedirs(vdir, exist_ok=True)
    cflags = [f for f in NVCC_FLAGS if f != "-shared"] + defs.split()

    def compile_one(src):
        obj = os.path.join(objdir, os.path.basename(src) + ".o")
        subprocess.check_call([nvcc] + cflags + ["-c", "-o", obj, src], cwd=CSRC)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        objs = list(ex.map(compile_one, sources()))
    out = os.path.join(vdir, f"libfpng_b200_{name}.so")
    subprocess.check_call([nvcc] + NVCC_FLAGS + ["-o", out + ".building"] + objs + LINK_FLAGS, cwd=CSRC)
    os.replace(out + ".building", out)
    return out


if __name__ == "__main__":
    print(build(force=True, verbose=True))
