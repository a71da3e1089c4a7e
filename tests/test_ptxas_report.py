"""The tensor-core query program compiles to asynchronous MMAs without local-memory traffic.

ptxas reports C7520 when it has to serialize a kernel's wgmma instructions (every MMA completes before the next
instruction, which removes the overlap the program is written for), and it reports the stack frame and the spill stores
and loads per kernel.  This test compiles query_tc.cu for sm_90a with the library's own flags and checks both, for every
instantiation of query_wg_kernel, query_jvp_kernel and g0_wg_kernel.  CPU only: it needs nvcc, not a GPU.
"""
import os
import re
import subprocess

import pytest

from monoport_b200 import build as lib_build

KERNELS = ("query_wg_kernel", "query_jvp_kernel", "g0_wg_kernel")


def _nvcc():
    try:
        return lib_build._nvcc()
    except RuntimeError:
        return None


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not available")
    out = tmp_path_factory.mktemp("ptxas") / "query_tc.o"
    cmd = [nvcc] + lib_build.NVCC_FLAGS + ["-c", os.path.join(lib_build.CSRC, "query_tc.cu"), "-o", str(out)]
    p = subprocess.run(cmd, capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    return p.stdout + p.stderr


def _entries(log):
    """{mangled kernel name: [its ptxas info lines]} for the kernels of KERNELS."""
    found = {}
    current = None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            current = m.group(1) if any(k in m.group(1) for k in KERNELS) else None
            if current:
                found[current] = []
        elif current and ("spill" in line or "registers" in line):
            found[current].append(line)
    return found


def test_each_head_has_a_plain_and_a_peer_store_instantiation(ptxas_log):
    names = list(_entries(ptxas_log))
    # query_wg_kernel: 2 heads x (plain, peer stores); query_jvp_kernel, g0_wg_kernel: 2 heads
    assert sum("query_wg_kernel" in n for n in names) == 4, names
    assert sum("query_jvp_kernel" in n for n in names) == 2, names
    assert sum("g0_wg_kernel" in n for n in names) == 2, names


def test_no_serialized_wgmma(ptxas_log):
    serialized = [line for line in ptxas_log.splitlines() if "C7520" in line and any(k in line for k in KERNELS)]
    assert not serialized, "\n".join(serialized)


def test_no_spills(ptxas_log):
    for name, lines in _entries(ptxas_log).items():
        stats = " ".join(lines)
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", stats)
        assert m, (name, stats)
        assert m.groups() == ("0", "0", "0"), (name, stats)
