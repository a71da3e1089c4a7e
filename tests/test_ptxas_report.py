"""The tensor-core query program compiles to asynchronous MMAs without local-memory traffic.

ptxas reports C7520 when it has to serialize a kernel's wgmma instructions (every MMA completes before the next
instruction, which removes the overlap the program is written for), and it reports the stack frame and the spill stores
and loads per kernel.  This test compiles query_tc.cu for sm_90a with the library's own flags and checks both, for every
instantiation of query_wg_kernel, query_jvp_kernel and g0_wg_kernel.  CPU only: it needs nvcc, not a GPU.
"""
import re

import pytest

from emu_harness import ptxas_report

KERNELS = ("query_wg_kernel", "query_jvp_kernel", "g0_wg_kernel")


@pytest.fixture(scope="module")
def report():
    """(the ptxas lines of the kernels of KERNELS by mangled name, the whole compiler output)"""
    entries, log = ptxas_report("query_tc.cu")
    return {name: lines for name, lines in entries if any(k in name for k in KERNELS)}, log


def test_each_head_has_a_plain_and_a_peer_store_instantiation(report):
    names = list(report[0])
    # query_wg_kernel: 2 heads x (plain, peer stores); query_jvp_kernel, g0_wg_kernel: 2 heads
    assert sum("query_wg_kernel" in n for n in names) == 4, names
    assert sum("query_jvp_kernel" in n for n in names) == 2, names
    assert sum("g0_wg_kernel" in n for n in names) == 2, names


def test_no_serialized_wgmma(report):
    serialized = [line for line in report[1].splitlines() if "C7520" in line and any(k in line for k in KERNELS)]
    assert not serialized, "\n".join(serialized)


def test_no_spills(report):
    for name, lines in report[0].items():
        stats = " ".join(lines)
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", stats)
        assert m, (name, stats)
        assert m.groups() == ("0", "0", "0"), (name, stats)
