"""Builds libglic_b200.so (the C-ABI CUDA library) and, optionally, the LibTorch shim, in-tree.

nvcc cross-compiles for sm_90a without a GPU.  Outputs (git-ignored):
  gaussian_lic_b200/libglic_b200.so        -- extern "C" ABI of include/glic_b200.h, no torch dependency
  gaussian_lic_b200/glic_b200_torch.so     -- reference operator symbols on top of the C ABI (torch_shim.cpp)
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
OBJ = os.path.join(PKG, "_build")
LIB = os.path.join(PKG, "libglic_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
HOST_CXX = "/usr/bin/g++"
CU_SOURCES = ["c_api.cu", "preprocess.cu", "radix_sort.cu", "render.cu", "preprocess_backward.cu", "ssim.cu", "adam_knn.cu", "p2p.cu", "model_step.cu", "map_io.cu", "extend.cu", "initialize.cu", "frames.cu", "lpips.cu", "prune.cu", "mesh.cu", "sparse_mesh.cu", "pose_correction.cu", "mapper.cu", "mapper_density.cu", "mapper_views.cu", "mapper_mesh.cu", "mapper_checkpoint.cu"]
NVCC_FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-ccbin", HOST_CXX,
              "-Xcompiler", "-fPIC,-fvisibility=hidden", "--expt-relaxed-constexpr"]


def _newer(target, deps):
    if not os.path.isfile(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def _headers():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hs.append(os.path.join(os.path.dirname(PKG), "include", "glic_b200.h"))
    return hs


def build_cuda(verbose=False, force=False):
    os.makedirs(OBJ, exist_ok=True)
    hdrs = _headers()
    jobs = []
    for src in CU_SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJ, src.replace(".cu", ".o"))
        if force or _newer(o, [s] + hdrs):
            cmd = [NVCC] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", s, "-o", o]
            jobs.append((src, cmd))

    def run(job):
        src, cmd = job
        p = subprocess.run(cmd, capture_output=True, text=True)
        return src, p.returncode, p.stdout + p.stderr

    with ThreadPoolExecutor(max_workers=8) as ex:
        for src, rc, out in ex.map(run, jobs):
            if verbose or rc:
                sys.stderr.write("== %s\n%s\n" % (src, out))
            if rc:
                raise RuntimeError("nvcc failed on %s" % src)
    objs = [os.path.join(OBJ, s.replace(".cu", ".o")) for s in CU_SOURCES]
    if force or jobs or _newer(LIB, objs):
        cmd = [NVCC, "-shared", "--cudart", "shared", "-ccbin", HOST_CXX, "-o", LIB] + objs
        subprocess.check_call(cmd)
    return LIB


TORCH_NAME = "glic_b200_torch"
TORCH_LIB = os.path.join(PKG, TORCH_NAME + ".so")


def build_torch_shim(verbose=False, force=False):
    """LibTorch shim (reference operator symbols + pybind face) linked against libglic_b200.so."""
    build_cuda(verbose=False)
    srcs = [os.path.join(CSRC, "torch_shim.cpp"), os.path.join(CSRC, "torch_shim_py.cpp"), os.path.join(CSRC, "torch_host.cpp")]
    if not force and not _newer(TORCH_LIB, srcs + _headers()):
        return TORCH_LIB
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
    os.environ["CXX"] = HOST_CXX
    from torch.utils import cpp_extension

    bdir = os.path.join(PKG, "_build_torch")
    os.makedirs(bdir, exist_ok=True)
    cpp_extension.load(
        name=TORCH_NAME, sources=srcs, extra_cflags=["-O2", "-std=c++17", "-w"],
        extra_include_paths=[cpp_extension.include_paths("cuda")[-1]] if False else [],
        # runpath relative to the library, so the tree can be built in one place and run in another: $ORIGIN for the copy in
        # PKG, $ORIGIN/.. for the one cpp_extension loads from _build_torch ($$ is ninja's escape, the quotes keep the shell
        # off it).  The SONAME lets a loaded shim satisfy the DT_NEEDED entry of oracle/_ref/glic_dropin_ext.so.
        extra_ldflags=["-L" + PKG, "-lglic_b200", "'-Wl,-rpath,$$ORIGIN:$$ORIGIN/..'", "-Wl,-soname," + TORCH_NAME + ".so"],
        with_cuda=True, build_directory=bdir, is_python_module=False, verbose=verbose)
    import shutil
    shutil.copy2(os.path.join(bdir, TORCH_NAME + ".so"), TORCH_LIB)
    return TORCH_LIB


if __name__ == "__main__":
    print(build_cuda(verbose="-v" in sys.argv, force="-f" in sys.argv))
    if "--torch" in sys.argv:
        print(build_torch_shim(verbose="-v" in sys.argv, force="-f" in sys.argv))
