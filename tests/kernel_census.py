"""Which CUDA kernels libfcsa_b200.so contains, and which ones a piece of host code launches.  Test infrastructure only.

`library_kernels` lists the library's __global__ instantiations from the ELF file, with binutils (readelf, nm,
c++filt) and no GPU.  nvcc registers every kernel of a module with the CUDA runtime by its mangled name: those
names are the C strings of .rodata that start with _Z.  They are cross-checked against the defined dynamic symbols
(each kernel has a host stub of the same mangled name), so a string that is not a kernel cannot slip in.

`launched_kernels` runs a callable under torch.profiler with CUDA activities and returns the library kernels that ran
on the device while it did.

Names are compared in one form: the demangled name without its return type and parameter list, e.g.
"fcsa::fcsa_fwd_kernel<__half, 64, false, true, true>".  The name builders below give that form from the template
arguments, in the template orders of the kernels:
    fcsa_fwd_kernel<T, D, BIAS, VARLEN, WINDOW>
    fcsa_bwd_kernel<T, D, BIAS, HEAD_LOOP, VARLEN, WINDOW, DQ>
    fcsa_dq_kernel<T, D, VARLEN, WINDOW>
    fcsa_decode_kernel<T, D, WINDOW>, decode_combine_kernel<T, D>
    bwd_prep_kernel<T, D / 8, VARLEN>, bwd_dq_finish_kernel<T, D, VARLEN>, bwd_kv_finish_kernel<T>
    row_fwd_kernel<T, X, TPR, U, APPEND>, row_bwd_kernel<T, X>  (X: the 16-bit type or float; TPR 4 / 8 for head
                                                                 dims 64 / 128, 0 for the others; U = 2)"""
import re
import shutil
import subprocess

import torch

# the family of each kernel template, in the order the census reports them
FAMILIES = {
    "fcsa_fwd_kernel": "forward",
    "fcsa_bwd_kernel": "backward",
    "fcsa_dq_kernel": "dQ",
    "fcsa_decode_kernel": "decode",
    "decode_combine_kernel": "combine",
    "bwd_prep_kernel": "prep",
    "bwd_dq_finish_kernel": "dq finish",
    "bwd_kv_finish_kernel": "kv finish",
    "varlen_tail_kernel": "varlen tail",
    "row_fwd_kernel": "row passes",
    "row_bwd_kernel": "row passes",
}


def _tool(name):
    path = shutil.which(name)
    assert path, f"{name} (binutils) not found on PATH"
    return path


def _run(cmd, stdin=None):
    # (readelf prints .rodata's binary data too: bytes that are not UTF-8 are replaced, names are ASCII)
    return subprocess.run(cmd, input=stdin, capture_output=True, text=True, errors="replace", check=True).stdout


def _params_start(name):
    """Index of the '(' that opens the parameter list of a demangled function name (outside every <...>)."""
    depth = 0
    for i, c in enumerate(name):
        if c == "<":
            depth += 1
        elif c == ">":
            depth -= 1
        elif c == "(" and depth == 0:
            return i
    return len(name)


def short_name(demangled):
    """'void fcsa::k<__half, 64, true>(CUtensorMap_st, ...)' -> 'fcsa::k<__half, 64, true>'"""
    name = demangled.strip()
    name = name[:_params_start(name)].strip()
    return name[len("void "):] if name.startswith("void ") else name


def family(name):
    base = name.split("<")[0].split("::")[-1]
    return FAMILIES.get(base)


def library_kernels(lib_path):
    """Sorted short names of every __global__ instantiation in the library."""
    rodata = _run([_tool("readelf"), "-p", ".rodata", lib_path])
    registered = sorted(set(re.findall(r"\]\s+(_Z\S+)", rodata)))
    defined = set()
    for line in _run([_tool("nm"), "-D", "--defined-only", lib_path]).splitlines():
        parts = line.split()
        if len(parts) == 3 and parts[1] in ("T", "W"):
            defined.add(parts[2])
    stray = [m for m in registered if m not in defined]
    assert not stray, f"registered names without a host stub: {stray}"
    demangled = _run([_tool("c++filt")], stdin="\n".join(registered) + "\n").splitlines()
    assert len(demangled) == len(registered)
    return sorted(short_name(d) for d in demangled)


def launched_kernels(fn):
    """Run fn() under torch.profiler (CUDA activities); returns (fn's result, the set of fcsa kernels that ran)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    names = set()
    for e in prof.events():
        if e.device_type.name == "CUDA":
            name = short_name(e.name)
            if name.startswith("fcsa::"):
                names.add(name)
    return out, names


# ---- names from template arguments ----------------------------------------------------------------------------------
_TYPES = {torch.bfloat16: "__nv_bfloat16", torch.float16: "__half", torch.float32: "float"}


def _arg(a):
    if isinstance(a, bool):
        return "true" if a else "false"
    if isinstance(a, torch.dtype):
        return _TYPES[a]
    return str(a)


def _k(base, *args):
    return f"fcsa::{base}<{', '.join(_arg(a) for a in args)}>"


def fwd(t, D, varlen=False, window=False, bias=False):
    return _k("fcsa_fwd_kernel", t, D, bias, varlen, window)


def bwd(t, D, head_loop=False, varlen=False, window=False, dq=True, bias=False):
    return _k("fcsa_bwd_kernel", t, D, bias, head_loop, varlen, window, dq)


def dq(t, D, varlen=False, window=False):
    return _k("fcsa_dq_kernel", t, D, varlen, window)


def decode(t, D, window=False):
    return _k("fcsa_decode_kernel", t, D, window)


def combine(t, D):
    return _k("decode_combine_kernel", t, D)


def prep(t, D, varlen=False):
    return _k("bwd_prep_kernel", t, D // 8, varlen)


def dq_finish(t, D, varlen=False):
    return _k("bwd_dq_finish_kernel", t, D, varlen)


def kv_finish(t):
    return _k("bwd_kv_finish_kernel", t)


VARLEN_TAIL = "fcsa::varlen_tail_kernel"


def row_fwd(t, D, x=None, append=False):
    """x: the input type (None: t, the 16-bit l2norm; torch.float32: the float32 cast)"""
    return _k("row_fwd_kernel", t, x or t, {64: 4, 128: 8}.get(D, 0), 2, append)


def row_bwd(t, x=None):
    return _k("row_bwd_kernel", t, x or t)
