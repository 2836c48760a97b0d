"""In-tree build of the engine's two binaries.

    libb200dpf.so                 CUDA kernels (sm_90a) + C ABI (include/b200dpf.h)
    dpf_cpp.<abi>.so              the `dpf_cpp` PyTorch extension module (pybind shim
                                  over the C ABI; same surface as the reference's
                                  dpf_wrapper.cu)

Both land next to this file so they travel to the GPU box with the gpurun
snapshot.  `python gpu-dpf_b200/build.py` builds whatever is stale.
"""
import os
import subprocess
import sys
import sysconfig

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
INCLUDE = os.path.join(ROOT, "include")

LIB = os.path.join(HERE, "libb200dpf.so")
EXT = os.path.join(HERE, "dpf_cpp" + (sysconfig.get_config_var("EXT_SUFFIX") or ".so"))

LIB_SOURCES = ["dpf_kernels.cu", "dpf_capi.cu", "dpf_plan.cu", "dpf_capi_keys.cu", "dpf_capi_multi.cu", "dpf_capi_group.cu",
               "dpf_capi_update.cu", "dpf_capi_batchcode.cu", "dpf_capi_kwpir.cu", "dpf_keygen.cu", "dpf_group_io.cu",
               "dpf_group_plan.cu", "dpf_batchcode.cu", "dpf_kwpir.cu", "dpf_host.cpp"]
# this script is a dependency too: its flags (the target architecture among them) shape both binaries
LIB_DEPS = LIB_SOURCES + ["dpf_core.cuh", "dpf_kernels.cuh", "dpf_host.h", "dpf_ctx.h", os.path.join(INCLUDE, "b200dpf.h"),
                          os.path.abspath(__file__)]
EXT_SOURCES = ["dpf_cpp_ext.cpp"]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC,-Wall,-Wno-unknown-pragmas",
]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    for d in deps:
        d = d if os.path.isabs(d) else os.path.join(CSRC, d)
        if os.path.getmtime(d) > t:
            return True
    return False


def build_lib(force=False, verbose=False):
    extra = os.environ.get("B200DPF_EXTRA_NVCC_FLAGS", "").split()
    cmd = [_nvcc()] + NVCC_FLAGS + extra + (["-Xptxas", "-v"] if verbose else []) + [
        "-shared", "-I", INCLUDE, "-o", LIB] + [os.path.join(CSRC, s) for s in LIB_SOURCES]
    # the command of the last build sits next to the library: a build with other flags (say, extra
    # ones from the environment) is not mistaken for an up-to-date one
    stamp = LIB + ".cmd"
    same_cmd = os.path.exists(stamp) and open(stamp).read() == " ".join(cmd)
    if not force and same_cmd and not _stale(LIB, LIB_DEPS):
        return LIB
    subprocess.run(cmd, check=True)
    with open(stamp, "w") as f:
        f.write(" ".join(cmd))
    return LIB


def build_ext(force=False):
    """Compile the pybind shim with g++ against torch's headers (host-only C++)."""
    build_lib(force=False)
    deps = EXT_SOURCES + [os.path.join(INCLUDE, "b200dpf.h"), os.path.abspath(__file__)]
    if not force and not _stale(EXT, deps):
        return EXT
    import torch
    from torch.utils import cpp_extension

    inc = []
    for p in cpp_extension.include_paths():
        inc += ["-isystem", p]
    inc += ["-isystem", sysconfig.get_paths()["include"], "-I", INCLUDE]
    torch_lib = os.path.join(os.path.dirname(torch.__file__), "lib")
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    cmd = ["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-unused-function",
           "-DTORCH_EXTENSION_NAME=dpf_cpp", "-DTORCH_API_INCLUDE_EXTENSION_H",
           "-D_GLIBCXX_USE_CXX11_ABI=%d" % abi] + inc + \
          [os.path.join(CSRC, s) for s in EXT_SOURCES] + \
          ["-o", EXT, "-L", HERE, "-lb200dpf", "-L", torch_lib, "-ltorch_python", "-ltorch", "-ltorch_cpu", "-lc10",
           "-Wl,-rpath,$ORIGIN", "-Wl,-rpath," + torch_lib]
    subprocess.run(cmd, check=True)
    return EXT


def build_all(force=False, verbose=False):
    build_lib(force=force, verbose=verbose)
    build_ext(force=force)


if __name__ == "__main__":
    build_all(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print("built:", LIB)
    print("built:", EXT)
