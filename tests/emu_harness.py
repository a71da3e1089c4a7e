"""The CPU model's plumbing, shared by the test modules: one g++ recipe for the harnesses of tests/emu (each compiled at most
once per pytest run), the writer of the query harnesses' in.bin (its layout: tests/emu/emu_host.h), and the ptxas report of a
library source compiled with the library's own flags."""
import functools
import os
import re
import shutil
import struct
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import spec

EMU = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
CUDA_INC = "/usr/local/cuda/include"
HAVE_GXX = shutil.which("g++") is not None
HAVE_CUDA_INC = os.path.exists(os.path.join(CUDA_INC, "cuda_fp16.h"))
needs_gxx = pytest.mark.skipif(not HAVE_GXX, reason="g++ not available")
needs_emu = pytest.mark.skipif(not (HAVE_GXX and HAVE_CUDA_INC), reason="g++ / CUDA headers not available")

# harness -> (optimisation level, includes the CUDA headers).  The query harnesses run 5-layer heads with one OS thread per
# CUDA thread: -O3 for the tensor-core programs and the gradient, -O2 for the other exact-kernel harnesses (their results
# are the same bits at every level: -ffp-contract=off and no fast-math); the integer / byte harnesses are light.
HARNESSES = {
    "emu_query_tc": ("-O3", True), "emu_query_jvp_tc": ("-O3", True), "emu_colour_surface_tc": ("-O3", True),
    "emu_dcal_tc": ("-O3", True), "emu_query_grad": ("-O3", True),
    "emu_query_fp32": ("-O2", True), "emu_heads_fp32": ("-O2", True), "emu_colour_surface_fp32": ("-O2", True),
    "emu_dcal_fp32": ("-O2", True),
    "emu_mcubes": ("-O1", False), "emu_mcubes_async": ("-O1", False), "emu_scan": ("-O1", False),
    "emu_octree": ("-O1", False), "emu_octree_loop": ("-O1", False), "emu_surface": ("-O1", False),
    "emu_display": ("-O1", False), "emu_render_normals": ("-O1", False),
}


def build(tmp_path_factory, name):
    """The executable of tests/emu/<name>.cpp, compiled on first use in this session (skips without g++ or, for the query
    harnesses, the CUDA headers)."""
    opt, cuda = HARNESSES[name]
    if not HAVE_GXX:
        pytest.skip("g++ not available")
    if cuda and not HAVE_CUDA_INC:
        pytest.skip("CUDA headers not found")
    exe = tmp_path_factory.getbasetemp() / "emu_bin" / name
    if not exe.exists():
        exe.parent.mkdir(exist_ok=True)
        # the kernels type-pun registers through reinterpret_cast like all CUDA code: no strict aliasing on the host build
        cmd = ["g++", "-std=c++17", opt, "-march=native", "-pthread", "-ffp-contract=off", "-Wno-unknown-pragmas",
               "-fno-strict-aliasing", "-DMP_CUDA_EMU=1", "-I" + CUDA_INC, "-I" + EMU, "-o", str(exe),
               os.path.join(EMU, name + ".cpp")]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
    return str(exe)


def write_input(path, feat, rows, calib, proj, res, last_op, Ws, bs, batched=False):
    """in.bin of the query harnesses.  feat [B,C,H,W]; rows [B,3,N] or [3,N] (points, or vertex rows X, Y, Z); calib [B,4,4]
    or None; Ws / bs the head's layers.  B = 1 unless batched (then B maps, point sets and calibs; otherwise the calib
    goes in the header)."""
    C, H, W = feat.shape[-3:]
    rows = np.ascontiguousarray(rows, dtype=np.float32)
    with open(path, "wb") as f:
        f.write(struct.pack("8i", C, H, W, rows.shape[-1], 1 if calib is not None else 0, 1 if proj == "perspective" else 0,
                            res, last_op))
        f.write(struct.pack("f", spec.Z_SCALE))
        head = calib[0, :3, :4].reshape(-1).tolist() if (calib is not None and not batched) else [0.0] * 12
        f.write(struct.pack("12f", *head))
        f.write(np.ascontiguousarray(feat, dtype=np.float32).tobytes())
        f.write(rows.tobytes())
        if batched and calib is not None:
            f.write(np.ascontiguousarray(calib[:, :3, :4], dtype=np.float32).tobytes())
        for Wl, bl in zip(Ws, bs):
            f.write(np.ascontiguousarray(Wl, dtype=np.float32).tobytes())
            f.write(np.ascontiguousarray(bl, dtype=np.float32).tobytes())


@functools.lru_cache(maxsize=None)
def _compile(nvcc, source):
    from monoport_b200 import build as lib_build
    with tempfile.TemporaryDirectory() as d:
        p = subprocess.run([nvcc] + lib_build.NVCC_FLAGS + ["-c", os.path.join(lib_build.CSRC, source), "-o",
                                                            os.path.join(d, "k.o")], capture_output=True, text=True)
    return p.returncode, p.stdout + p.stderr


def ptxas_report(source):
    """monoport_b200/csrc/<source> compiled for sm_90a with the library's flags, once per session (skips without nvcc).
    -> (entries, log): entries = [(mangled kernel name, [its ptxas lines: stack frame and spills, registers])] in the order
    ptxas compiled them; log = the whole compiler output."""
    from monoport_b200 import build as lib_build
    try:
        nvcc = lib_build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not available")
    rc, log = _compile(nvcc, source)
    assert rc == 0, log
    entries, current = [], None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            current = (m.group(1), [])
            entries.append(current)
            continue
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            if current and m.group(1) != current[0]:
                current = None                  # a non-entry function's report
        elif current and ("stack frame" in line or "registers" in line):
            current[1].append(line)
    return entries, log
