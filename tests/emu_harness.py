"""The CPU model's plumbing, shared by the test modules: one g++ recipe for the harnesses of tests/emu (each compiled at most
once per pytest run), the writer of the query harnesses' in.bin (its layout: tests/emu/emu_host.h), one runner of the query
harnesses, and the ptxas report of a library source compiled with the library's own flags."""
import functools
import os
import pathlib
import re
import shutil
import struct
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from oracle import spec

EMU = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
CUDA_INC = "/usr/local/cuda/include"
HAVE_GXX = shutil.which("g++") is not None
HAVE_CUDA_INC = os.path.exists(os.path.join(CUDA_INC, "cuda_fp16.h"))
needs_gxx = pytest.mark.skipif(not HAVE_GXX, reason="g++ not available")
needs_emu = pytest.mark.skipif(not (HAVE_GXX and HAVE_CUDA_INC), reason="g++ / CUDA headers not available")

# harness -> (optimisation level, includes the CUDA headers).  The query harnesses run 5-layer heads with one OS thread per
# CUDA thread: -O3 (their results are the same bits at every level: -ffp-contract=off and no fast-math); the integer /
# byte harnesses are light.
HARNESSES = {
    "emu_tc": ("-O3", True), "emu_fp32": ("-O3", True),
    "emu_mcubes": ("-O1", False), "emu_mcubes_async": ("-O1", False), "emu_scan": ("-O1", False),
    "emu_octree": ("-O1", False), "emu_octree_loop": ("-O1", False), "emu_surface": ("-O1", False),
    "emu_display": ("-O1", False), "emu_render_normals": ("-O1", False),
}


def build(tmp_path_factory, name):
    """The executable of tests/emu/<name>.cpp, compiled on first use in this session (skips without g++ or, for the query
    harnesses, the CUDA headers).  tmp_path_factory: pytest's, or a directory to build into."""
    opt, cuda = HARNESSES[name]
    if not HAVE_GXX:
        pytest.skip("g++ not available")
    if cuda and not HAVE_CUDA_INC:
        pytest.skip("CUDA headers not found")
    if isinstance(tmp_path_factory, (str, pathlib.Path)):
        exe = pathlib.Path(tmp_path_factory) / name
    else:
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


def _side_file(path, x):
    np.ascontiguousarray(x.numpy() if isinstance(x, torch.Tensor) else x, dtype=np.float32).tofile(path)
    return str(path)


def run(exe, tmp_path, op, *args, inp, shape, options=None, env=None, tag="x", returncode=0):
    """One run of a query harness (tests/emu/emu_fp32.cpp or emu_tc.cpp): in.bin = write_input(**inp), then
    `exe in.bin out.f32 op args --options`.  An array among args, or as an option's value, goes to a side file (a
    grad_output, a --dcal camera) whose path takes its place.  options: {name: value} (canvas_bg for --canvas-bg), True
    for a flag, None / False to leave it out.  env: the model's own knobs (EMU_TC_ORDER ...).  tag keeps the files of
    several runs in one tmp_path apart.
    -> (out, the finished process): out = out.f32 as a float32 tensor of `shape` (shape None: its raw bytes; None when
    the harness is expected to fail with `returncode`)."""
    fin, fout = tmp_path / ("in_%s.bin" % tag), tmp_path / ("out_%s.f32" % tag)
    write_input(fin, **inp)
    argv = [exe, str(fin), str(fout), op]
    for i, a in enumerate(args):
        is_array = isinstance(a, (np.ndarray, torch.Tensor))
        argv.append(_side_file(tmp_path / ("arg%d_%s.f32" % (i, tag)), a) if is_array else str(a))
    for k, v in (options or {}).items():
        if isinstance(v, (np.ndarray, torch.Tensor)):
            v = _side_file(tmp_path / ("%s_%s.f32" % (k, tag)), v)
        if v is True:
            argv.append("--" + k.replace("_", "-"))
        elif v is not None and v is not False:
            argv.append("--%s=%s" % (k.replace("_", "-"), v))
    if fout.exists():
        fout.unlink()
    r = subprocess.run(argv, capture_output=True, text=True, timeout=3600, env=dict(os.environ, **(env or {})))
    assert r.returncode == returncode and "DEADLOCK" not in r.stderr, r.stderr[-2000:]
    if returncode:
        return None, r
    if shape is None:
        return fout.read_bytes(), r
    out = np.fromfile(fout, dtype=np.float32)
    assert out.size == int(np.prod(shape)), (out.size, shape)
    return torch.from_numpy(out).reshape(shape), r


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
