"""The implicit-GEMM and weight-gradient kernels keep every value in registers: no stack frame, no spill, no local-memory
instruction. Their shared-memory rings leave L1 little room, so local memory would go to L2 on the critical path.
`meshdiffusion_b200/build.py` fails a build whose ptxas report shows otherwise; these tests check that guard on canned
reports and the built library's SASS."""
import os
import re
import shutil
import subprocess

import pytest

CLEAN = """\
ptxas info    : Compiling entry function '_ZN3mdb14gemm_tc_kernelILi128ELNS_9PrecisionE2ELb0EEEvNS_10GemmParamsE' for 'sm_90a'
ptxas info    : Function properties for _ZN3mdb14gemm_tc_kernelILi128ELNS_9PrecisionE2ELb0EEEvNS_10GemmParamsE
    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads
ptxas info    : Used 168 registers, used 3 barriers
ptxas info    : Function properties for _ZN3mdb19pack_weights_kernelILNS_9PrecisionE0EEEvPKNS_9LoadEntryEPKiiNS_8PackArgsEiiiPv
    64 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads
"""


def _report(fn, stack, spill_st, spill_ld):
    return (f"ptxas info    : Function properties for {fn}\n"
            f"    {stack} bytes stack frame, {spill_st} bytes spill stores, {spill_ld} bytes spill loads\n")


def test_guard_passes_a_clean_report_and_other_kernels():
    from meshdiffusion_b200 import build
    assert build.local_memory_violations(CLEAN) == []


@pytest.mark.parametrize("fn", ["_ZN3mdb14gemm_tc_kernelILi32ELNS_9PrecisionE0ELb1EEEvNS_10GemmParamsE",
                                "_ZN3mdb15wgrad_tc_kernelILNS_9PrecisionE2EEEvNS_11WgradParamsE"])
@pytest.mark.parametrize("frame", [(256, 0, 0), (0, 8, 0), (0, 0, 8)])
def test_guard_flags_stack_and_spills(fn, frame):
    from meshdiffusion_b200 import build
    bad = build.local_memory_violations(CLEAN + _report(fn, *frame))
    assert len(bad) == 1 and bad[0].startswith(fn)


def test_built_kernels_have_no_local_memory_instructions():
    from meshdiffusion_b200 import _native
    _native.lib()
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", _native.LIB_PATH], capture_output=True, text=True, check=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)[1:]
    checked = 0
    for f in funcs:
        name = f.split("\n", 1)[0].strip()
        if not any(k in name for k in ("gemm_tc_kernel", "wgrad_tc_kernel")):
            continue
        checked += 1
        local = re.findall(r"\b(STL|LDL)(\.\w+)*\b", f)
        assert not local, f"{name}: {len(local)} local-memory instructions"
    assert checked >= 12  # 10 implicit-GEMM instantiations + 2 weight-gradient ones
