"""CPU: what ptxas reported when it compiled libfcsa_b200.so (the `-Xptxas -v` output that build.py keeps in
flash_cosine_sim_attention_b200/build.log).  Skipped when there is no log (a library built some other way).

* No kernel of the library may have its wgmmas serialised.  ptxas does that silently, with only an info note
  (C7510 - C7520, "wgmma.mma_async instructions are serialized ..."), when it runs out of registers or cannot prove a
  register an asynchronous wgmma reads or writes is left alone; the kernel then runs far slower (DESIGN.md 4.2: the
  backward took 629 instead of 435 us) and computes the same results, so no parity test sees it.
* The D = 64 backward kernels with three key warpgroups run their consumers at 160 registers, where a few loop-invariant
  scalars spill.  Their spill stores may not grow past a pinned budget per instantiation."""
import os
import re
import subprocess

import pytest

from flash_cosine_sim_attention_b200.build import LOG
from kernel_census import _tool, bwd, short_name

# spill-store bytes allowed per wide backward instantiation (the figures of the 192-key kernels when they were
# introduced; fcsa_bwd_kernel<T, 64, BIAS = false, HEAD_LOOP = false, VARLEN, WINDOW, DQ = true>)
WIDE_SPILL_BUDGET = {(False, False): 44, (True, False): 56, (False, True): 68, (True, True): 60}
WIDE_KERNELS = {bwd(t, 64, varlen=v, window=w): budget
                for t in ("__half", "__nv_bfloat16") for (v, w), budget in WIDE_SPILL_BUDGET.items()}

_ENTRY = re.compile(r"Compiling entry function '(_Z\S+)'")
_PROPS = re.compile(r"Function properties for (_Z\S+)")
_SPILL = re.compile(r"(\d+) bytes spill stores")
_NOTE_FN = re.compile(r"function '(_Z[^']+)'")


def parse_log(text):
    """{short kernel name: {"spill_stores": bytes, "notes": [ptxas notes naming the kernel]}} of every kernel."""
    per, cur = {}, None
    for line in text.splitlines():
        m = _ENTRY.search(line)
        if m:
            per.setdefault(m.group(1), {"spill_stores": None, "notes": []})
            continue
        m = _PROPS.search(line)
        if m:
            cur = m.group(1)
            per.setdefault(cur, {"spill_stores": None, "notes": []})
            continue
        m = _SPILL.search(line)
        if m and cur is not None:
            per[cur]["spill_stores"] = int(m.group(1))
            cur = None
            continue
        m = _NOTE_FN.search(line)
        if m:
            per.setdefault(m.group(1), {"spill_stores": None, "notes": []})["notes"].append(line.strip())
    mangled = sorted(per)
    out = subprocess.run([_tool("c++filt")], input="\n".join(mangled) + "\n", capture_output=True, text=True,
                         check=True).stdout.splitlines()
    assert len(out) == len(mangled)
    return {short_name(d): per[m] for m, d in zip(mangled, out)}


def serialises_wgmma(note):
    return "wgmma" in note and "serializ" in note


@pytest.fixture(scope="module")
def kernels():
    if not os.path.exists(LOG):
        pytest.skip("no build log next to the library: build it with flash_cosine_sim_attention_b200.build")
    with open(LOG) as f:
        per = parse_log(f.read())
    if not any(k.startswith("fcsa::") for k in per):
        pytest.skip("the build log holds no ptxas output for the library's kernels")
    return per


def test_parse_log():
    name = "_ZN4fcsa15fcsa_bwd_kernelI6__halfLi64ELb0ELb0ELb0ELb0ELb1EEEvv"
    text = (f"ptxas info    : Compiling entry function '{name}' for 'sm_90a'\n"
            f"ptxas info    : Function properties for {name}\n"
            "    24 bytes stack frame, 44 bytes spill stores, 40 bytes spill loads\n"
            "ptxas info    : (C7512) Potential Performance Loss: wgmma.mma_async instructions are serialized due to "
            f"insufficient register resources for the function '{name}'\n")
    per = parse_log(text)
    k = per["fcsa::fcsa_bwd_kernel<__half, 64, false, false, false, false, true>"]
    assert k["spill_stores"] == 44
    assert len(k["notes"]) == 1 and serialises_wgmma(k["notes"][0])
    assert not serialises_wgmma("ptxas info    : (C7519) warpgroup.arrive is injected in around line 1 by compiler "
                                "to allow use of registers in GMMA in function 'x'")


def test_no_serialised_wgmma(kernels):
    bad = {k: [n for n in v["notes"] if serialises_wgmma(n)] for k, v in kernels.items()}
    bad = {k: n for k, n in bad.items() if n}
    assert not bad, "ptxas serialised the wgmmas of: " + "; ".join(f"{k}: {n[0]}" for k, n in sorted(bad.items()))


def test_wide_backward_spill_budget(kernels):
    missing = [k for k in WIDE_KERNELS if k not in kernels or kernels[k]["spill_stores"] is None]
    assert not missing, f"no ptxas figures in the build log for {missing}"
    over = {k: kernels[k]["spill_stores"] for k, budget in WIDE_KERNELS.items() if kernels[k]["spill_stores"] > budget}
    print({k: kernels[k]["spill_stores"] for k in sorted(WIDE_KERNELS)})
    assert not over, f"spill stores over budget {WIDE_SPILL_BUDGET}: {over}"
