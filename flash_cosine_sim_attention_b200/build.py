"""Builds the two native artefacts in-tree, for sm_90a (H100) only:

  libfcsa_b200.so                                  the C-ABI CUDA library (nvcc, one -gencode)
  flash_cosine_sim_attention_cuda_0_1_40.*.so      the PyTorch extension module over that ABI (host C++
                                                   compiler only) - the module the reference builds with
                                                   its setup.py CUDAExtension (setup.py:30-39, no arch flags
                                                   there) and imports by this versioned name (version.py:3)

    python -m flash_cosine_sim_attention_b200.build        # build (skips what is up to date)
    python -m flash_cosine_sim_attention_b200.build -f     # force rebuild

The repository's setup.py drives the same two steps for `pip install .` / `build_ext --inplace`.
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
ROOT = os.path.dirname(HERE)
LIB = os.path.join(HERE, "libfcsa_b200.so")
# the command line and the compiler output of the last library build: -Xptxas -v gives every kernel's registers and
# spills, and ptxas notes there when it serialises a kernel's wgmmas (tests/test_ptxas_log.py reads it)
LOG = os.path.join(HERE, "build.log")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "--shared", "-Xcompiler", "-fPIC",
    "-Xptxas", "-v",
    "--expt-relaxed-constexpr",
]


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: libfcsa_b200.so cannot be built")


def _sources():
    return [os.path.join(CSRC, "fcsa_abi.cu")]


def _deps():
    out = [os.path.join(ROOT, "include", "fcsa_b200.h")]
    for f in sorted(os.listdir(CSRC)):
        if f.endswith((".cu", ".cuh", ".h")):
            out.append(os.path.join(CSRC, f))
    return out


# ---- the torch extension module ---------------------------------------------------------------------
EXT_NAME = "flash_cosine_sim_attention_cuda_0_1_40"     # reference version.py:3 (__cuda_pkg_name__)
EXT_SRC = os.path.join(CSRC, "torch_ext.cpp")


def ext_path():
    import sysconfig
    return os.path.join(HERE, EXT_NAME + sysconfig.get_config_var("EXT_SUFFIX"))


def ext_compile_command(out=None):
    """The g++ command line (list) that builds the extension module next to libfcsa_b200.so."""
    import sysconfig
    import torch
    from torch.utils import cpp_extension as ce
    cuda_home = os.environ.get("CUDA_HOME") or os.path.dirname(os.path.dirname(_nvcc()))
    inc = list(ce.include_paths()) + [os.path.join(cuda_home, "include"), sysconfig.get_paths()["include"]]
    libdirs = list(ce.library_paths()) + [os.path.join(cuda_home, "lib64")]
    # the system g++ on PATH, as nvcc uses for the library.  ($CXX in this image points at a wrapped toolchain
    # under /opt/gcc whose objects crash while unwinding a c10::Error through pybind11 - measured here; set
    # FCSA_CXX to override)
    cxx = os.environ.get("FCSA_CXX") or shutil.which("g++") or "g++"
    cmd = [cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-fvisibility=hidden", "-Wall", "-Wno-unused-function",
           f"-DTORCH_EXTENSION_NAME={EXT_NAME}", "-DTORCH_API_INCLUDE_EXTENSION_H",
           f"-D_GLIBCXX_USE_CXX11_ABI={int(torch._C._GLIBCXX_USE_CXX11_ABI)}"]
    cmd += [f"-I{d}" for d in inc]
    cmd += [EXT_SRC, "-o", out or ext_path()]
    cmd += [f"-L{d}" for d in libdirs] + [f"-L{HERE}", "-l:libfcsa_b200.so"]
    cmd += ["-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch", "-ltorch_python", "-lcudart"]
    # $ORIGIN: in-tree (module next to the library); $ORIGIN/<package>: pip-installed (module top-level)
    cmd += ["-Wl,-rpath,$ORIGIN", "-Wl,-rpath,$ORIGIN/flash_cosine_sim_attention_b200"]
    cmd += [f"-Wl,-rpath,{d}" for d in ce.library_paths()]
    return cmd


def ext_up_to_date():
    out = ext_path()
    if not os.path.exists(out):
        return False
    t = os.path.getmtime(out)
    return all(os.path.getmtime(d) <= t for d in (EXT_SRC, os.path.join(ROOT, "include", "fcsa_b200.h")))


def build_extension(force=False, verbose=False):
    """Compile the torch extension module if needed (needs libfcsa_b200.so next to it); returns its path."""
    build_library(force=False)
    if not force and ext_up_to_date():
        return ext_path()
    cmd = ext_compile_command()
    proc = subprocess.run(cmd, capture_output=True, text=True)
    log = proc.stdout + proc.stderr
    with open(os.path.join(HERE, "build_ext.log"), "w") as f:
        f.write(" ".join(cmd) + "\n" + log)
    if proc.returncode != 0:
        raise RuntimeError("extension build failed:\n" + log[-8000:])
    if verbose:
        print(log)
    return ext_path()


def up_to_date():
    if not os.path.exists(LIB):
        return False
    t = os.path.getmtime(LIB)
    return all(os.path.getmtime(d) <= t for d in _deps())


def build_library(force=False, verbose=False):
    """Compile the library if needed; returns its path."""
    if not force and up_to_date():
        return LIB
    cmd = [_nvcc()] + NVCC_FLAGS + ["-o", LIB] + _sources()
    proc = subprocess.run(cmd, capture_output=True, text=True)
    log = proc.stdout + proc.stderr
    with open(LOG, "w") as f:
        f.write(" ".join(cmd) + "\n" + log)
    if proc.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + log[-8000:])
    if verbose:
        print(log)
    return LIB


if __name__ == "__main__":
    print(build_library(force="-f" in sys.argv, verbose="-v" in sys.argv))
    print(build_extension(force="-f" in sys.argv, verbose="-v" in sys.argv))
