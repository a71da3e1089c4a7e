"""CPU tier of the display images (visulization, RTL/main.py:252-281): display_kernel compiled unmodified against the CPU
emulation layer (tests/emu) on 1-3 CTAs, bit for bit against the reference's own outputs (tests/golden/display_*.npz) and
against the restatement display_cases.visulization_ref over the downscale, identity, x2 and general nearest paths; the
compiler report of the kernel; and the refusals of mp_display_async that need no device."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from display_cases import display_canvases, visulization_ref

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu")
GOLDEN = os.path.join(HERE, "golden")
CUDA_INC = "/usr/local/cuda/include"
S = 256

emu_available = pytest.mark.skipif(shutil.which("g++") is None or not os.path.exists(os.path.join(CUDA_INC, "cuda_fp16.h")),
                                   reason="g++ / CUDA headers not available")


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("emu_display") / "emu_display")
    cmd = ["g++", "-std=c++17", "-pthread", "-ffp-contract=off", "-Wno-unknown-pragmas", "-fno-strict-aliasing", "-O1",
           "-DMP_CUDA_EMU=1", "-I" + CUDA_INC, "-I" + EMU, "-o", exe, os.path.join(EMU, "emu_display.cpp")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return exe


def _display(exe, tmp_path, norm, tex, blocks, size=S):
    """display_kernel on the CPU model -> (norm [size,size,3] or None, tex likewise, mask [size,size,1] bool)"""
    R = (norm if norm is not None else tex).shape[0]
    images = "both" if norm is not None and tex is not None else ("norm" if tex is None else "tex")
    fin, fout = str(tmp_path / "d.bin"), str(tmp_path / "d.out")
    with open(fin, "wb") as f:
        for c in (norm, tex):
            if c is not None:
                f.write(np.ascontiguousarray(c, dtype=np.float32).tobytes())
    r = subprocess.run([exe, str(R), str(size), str(blocks), images, fin, fout], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    raw = np.fromfile(fout, dtype=np.uint8)
    n3 = size * size * 3 * 4
    out, off = [], 0
    for c in (norm, tex):
        if c is None:
            out.append(None)
        else:
            out.append(raw[off:off + n3].view(np.float32).reshape(size, size, 3))
            off += n3
    mask = raw[off:]
    assert mask.size == size * size and set(np.unique(mask)) <= {0, 1}
    return out[0], out[1], mask.astype(bool).reshape(size, size, 1)


def _same(a, b):
    """bit for bit (NaN payloads included) for images, equal for masks; None only against None"""
    if a is None or b is None:
        return a is None and b is None
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    if a.dtype == np.float32:
        return a.shape == b.shape and b.dtype == np.float32 and np.array_equal(a.view(np.int32), b.view(np.int32))
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a, b)


def _golden(R):
    return np.load(os.path.join(GOLDEN, "display_%d.npz" % R))


CASES = ["both", "norm", "tex"]


def _case_inputs(norm, tex, case):
    return (norm if case != "tex" else None), (tex if case != "norm" else None)


def _golden_want(g, case):
    mask = {"both": g["mask_both"], "norm": g["mask_norm"], "tex": g["mask_tex"]}[case]
    return (g["render_norm"] if case != "tex" else None), (g["render_tex"] if case != "norm" else None), mask


# ---- the kernel against the reference's outputs ------------------------------------------------------------------------
@emu_available
@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("R", [257, 129, 33])
def test_kernel_matches_reference_goldens(emu, tmp_path, R, case):
    """The unmodified reference visulization's outputs: images bit for bit (NaN included) and the mask, for both images and
    for each image alone, on 1, 2 and 3 CTAs."""
    g = _golden(R)
    want = _golden_want(g, case)
    for blocks in (1, 2, 3):
        got = _display(emu, tmp_path, *_case_inputs(g["norm"], g["tex"], case), blocks)
        for k, (a, b) in enumerate(zip(got, want)):
            assert _same(a, b), (R, case, blocks, k)


def test_goldens_cover_the_edge_values():
    """The goldens hold what the kernel must get right: NaN outputs, pixels with only one or two channels at 255, a texture
    background that is not white, and a mask that differs between the normal and the texture image."""
    for R in (257, 129, 33):
        g = _golden(R)
        for img in (g["render_norm"], g["render_tex"]):
            assert np.isnan(img).any()
            full = (img == 255).sum(axis=2)
            assert ((full == 1) | (full == 2)).any() and (full == 3).any()
        assert (g["tex"] == 0.75).all(axis=2).any()
        assert np.array_equal(g["mask_both"], g["mask_tex"]) and not np.array_equal(g["mask_both"], g["mask_norm"])
        assert (g["mask_tex"] & ~g["mask_norm"]).any() and (g["mask_norm"] & ~g["mask_tex"]).any()


@pytest.mark.parametrize("R", [257, 129, 33])
def test_restatement_matches_reference_goldens(R):
    g = _golden(R)
    norm, tex = torch.from_numpy(g["norm"]), torch.from_numpy(g["tex"])
    for case in CASES:
        got = visulization_ref(*_case_inputs(norm, tex, case))
        for k, (a, b) in enumerate(zip(got, _golden_want(g, case))):
            assert _same(a, b), (R, case, k)
    assert visulization_ref(None, None) == (None, None, None)


# ---- the kernel against the restatement over every nearest path ----------------------------------------------------------
@emu_available
@pytest.mark.parametrize("R,size", [(17, S), (33, S), (128, S), (129, S), (256, S), (257, S), (513, S), (33, 100)])
def test_kernel_matches_restatement(emu, tmp_path, R, size):
    """Downscale (513, 257), identity (256), x2 (128) and general nearest upscales, each case on its own CTA count: bit for
    bit, and the mask from the texture image whenever it is present."""
    norm, tex = display_canvases(R, 100 + R)
    for i, case in enumerate(CASES):
        n, t = _case_inputs(norm, tex, case)
        want = visulization_ref(n, t, size=size)
        got = _display(emu, tmp_path, None if n is None else n.numpy(), None if t is None else t.numpy(), 1 + i, size)
        for k, (a, b) in enumerate(zip(got, want)):
            assert _same(a, b), (R, size, case, k)
        if case == "both":
            assert np.array_equal(got[2], visulization_ref(None, t, size=size)[2])
            assert not np.array_equal(got[2], visulization_ref(n, None, size=size)[2])


# ---- compiler report ---------------------------------------------------------------------------------------------------
def test_display_kernel_has_no_frame_and_no_spills(tmp_path):
    from monoport_b200 import build as lib_build
    try:
        nvcc = lib_build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not available")
    p = subprocess.run([nvcc] + lib_build.NVCC_FLAGS + ["-c", os.path.join(lib_build.CSRC, "surface.cu"), "-o",
                                                        str(tmp_path / "surface.o")], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    log = (p.stdout + p.stderr).splitlines()
    at = [i for i, line in enumerate(log) if re.search(r"Compiling entry function '\w*display_kernel\w*'", line)]
    assert len(at) == 1, at
    stats = " ".join(log[at[0]:at[0] + 4])
    assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in stats, stats


# ---- the C ABI: refusals before any device work ------------------------------------------------------------------------
def test_abi_refusals_that_need_no_device():
    """mp_display_async refuses NULL for both images, R < 1, S < 1, a missing output of a present image, and a NULL mask
    or staging buffer -- before any CUDA call, so these hold on a machine without a GPU."""
    from monoport_b200 import _lib, build
    build.build()
    lib = _lib.load()
    dev = ctypes.c_void_p(0x1000)           # never dereferenced: every call below is refused first
    host = ctypes.c_void_p(0x2000)

    def call(norm=dev, tex=dev, R=33, size=S, norm_host=host, tex_host=host, mask=host, staging=dev):
        return lib.mp_display_async(norm, tex, R, size, norm_host, tex_host, mask, staging, None)

    cases = {"both images NULL": dict(norm=None, tex=None), "R = 0": dict(R=0), "R < 0": dict(R=-5), "S = 0": dict(size=0),
             "no normal output": dict(norm_host=None), "no texture output": dict(tex_host=None),
             "no texture output (texture only)": dict(norm=None, norm_host=None, tex_host=None),
             "no mask": dict(mask=None), "no staging": dict(staging=None)}
    for what, kw in cases.items():
        assert call(**kw) == -1, what
        assert lib.mp_last_error(), what
    call(norm=None, tex=None)
    assert b"both images are NULL" in lib.mp_last_error()
