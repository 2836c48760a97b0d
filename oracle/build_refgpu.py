"""Build the UNMODIFIED reference GPU extension for sm_90a -- TEST INFRASTRUCTURE ONLY.

Compiles /root/reference/dpf_wrapper.cu (which #includes dpf_base/dpf.h and
dpf_gpu/dpf/dpf_hybrid.cu) where it lies, with one nvcc command of ours (the
reference's setup.py is not run), into oracle/_ref/ref_dpf_cpp.so -- the
reference's `dpf_cpp` pybind module under the name `ref_dpf_cpp` so it can be
imported next to ours.  Used for (1) a second parity check, GPU kernel against
GPU kernel, and (2) the "reference kernel on the same H100" column of
DESIGN.md / profiles.  Needs the reference tree, so it only runs in the build
container; the .so travels to the GPU box with the gpurun snapshot.
"""
import os
import subprocess
import sys
import sysconfig

HERE = os.path.dirname(os.path.abspath(__file__))
REF_ROOT = os.environ.get("REF_ROOT", "/root/reference")
OUT = os.path.join(HERE, "_ref", "ref_dpf_cpp.so")


def build(force=False):
    src = os.path.join(REF_ROOT, "dpf_wrapper.cu")
    if not os.path.exists(src):
        print("reference tree %s absent: keeping prebuilt oracle/_ref/ref_dpf_cpp.so (if any)" % REF_ROOT)
        return None
    # this script's flags (the target architecture among them) shape the binary too
    if not force and os.path.exists(OUT) and os.path.getmtime(OUT) >= max(os.path.getmtime(src), os.path.getmtime(__file__)):
        return OUT
    import torch
    from torch.utils import cpp_extension
    inc = []
    for p in cpp_extension.include_paths():
        inc += ["-isystem", p]
    inc += ["-isystem", sysconfig.get_paths()["include"]]
    tl = os.path.join(os.path.dirname(torch.__file__), "lib")
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    cmd = ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-shared",
           "-Xcompiler", "-fPIC", "-w", "-DTORCH_EXTENSION_NAME=ref_dpf_cpp", "-DTORCH_API_INCLUDE_EXTENSION_H",
           "-D_GLIBCXX_USE_CXX11_ABI=%d" % int(torch._C._GLIBCXX_USE_CXX11_ABI), "-I", REF_ROOT] + inc + \
          [src, "-o", OUT, "-L", tl, "-ltorch_python", "-ltorch", "-ltorch_cpu", "-ltorch_cuda", "-lc10", "-lc10_cuda",
           "-Xlinker", "-rpath," + tl]
    subprocess.run(cmd, check=True)
    print("built", OUT, "from", src)
    return OUT


if __name__ == "__main__":
    build(force="--force" in sys.argv)
