"""CPU tier of the per-frame camera: every program a captured frame launches, compiled unmodified against the CPU emulation
layer (tests/emu), reads its camera from device memory (a single-map MpBatch whose calibs point at a 12-float buffer, the
EMU_DCAL flag of tests/emu/emu_dcal_fp32.cpp and emu_dcal_tc.cpp) and must give, bit for bit, what its by-value launch gives with the same 12 floats -- the exact
query over a node list with the volume scatter, the tensor-core query over a node list and over a grid range, the colour
surface render of both programs, and both gradient programs.  Every case runs two launches through one buffer rewritten
between them, and each must give its own camera's result."""
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import spec
from emu_harness import build, needs_emu, write_input
from grad_cases import load_grad_case

pytestmark = needs_emu

R = 65
UNIT = ["-1", "-1", "-1", "1", "1", "1"]


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return {k: build(tmp_path_factory, "emu_dcal_" + k) for k in ("fp32", "tc")}


def _case(name, proj):
    """a golden's head, map and points, with the projection asked for"""
    c = dict(load_grad_case(name))
    c["proj"] = proj
    return c


def _second_camera(c):
    """another camera for the same scene: the demo's at a different pitch (perspective cases: the golden's, turned)"""
    if c["proj"] == "perspective":
        cal = c["calib"].clone()
        cal[0, :3, :3] = cal[0, :3, :3] @ torch.tensor([[0.0, 0.0, 1.0], [0.0, 1.0, 0.0], [-1.0, 0.0, 0.0]])
        return cal
    return spec.scene_calib(20, 63)


def _write(path, c, rows, calib=None):
    """in.bin of the harnesses: header, z_scale, calib rows 0..2, the map, three rows of N floats, the head"""
    write_input(path, c["feat"], rows, c["calib"] if calib is None else calib, c["proj"], c["chans"][-1], c["last_op"], c["Ws"],
                c["bs"])


def _run(tmp_path, tag, exe, args, c, rows, env=None):
    """the by-value launches with camera A (the case's) and camera B, and the device-calib pair (B, then A) through one
    buffer -> the four outputs as raw float32 arrays"""
    cal_b = _second_camera(c)
    fa, fb = (str(tmp_path / ("%s_%s.bin" % (tag, k))) for k in "ab")
    _write(fa, c, rows)
    _write(fb, c, rows, cal_b)
    first = str(tmp_path / ("%s_first.f32" % tag))
    np.asarray(cal_b[0, :3, :4].reshape(-1).tolist(), dtype=np.float32).tofile(first)
    outs = {}
    for key, fin, extra in (("a", fa, {}), ("b", fb, {}), ("d", fa, {"EMU_DCAL": first})):
        fout = str(tmp_path / ("%s_out_%s.f32" % (tag, key)))
        r = subprocess.run([exe, fin, fout] + args, capture_output=True, text=True, timeout=3600,
                           env=dict(os.environ, **(env or {}), **extra))
        assert r.returncode == 0 and "DEADLOCK" not in r.stderr, r.stderr[-2000:]
        outs[key] = np.fromfile(fout, dtype=np.float32)
        if key == "d":
            outs["d_first"] = np.fromfile(fout + ".first", dtype=np.float32)
    return outs


def _assert_bits(outs, min_distinct=1):
    a, b = outs["a"], outs["b"]
    assert a.tobytes() == outs["d"].tobytes(), "device calib (A, after the buffer was rewritten) != by-value A"
    assert b.tobytes() == outs["d_first"].tobytes(), "device calib (B, first launch) != by-value B"
    # the two cameras see different things: a launch that ignored the buffer could not pass both checks
    assert int((a.view(np.uint32) != b.view(np.uint32)).sum()) >= min_distinct


def _points(c, n):
    return c["points"][0, :, :n].numpy()


# ---- the exact kernel over a node list with the volume scatter (the octree engine's fused path) ---------------------------
@pytest.mark.parametrize("proj,sms", [("orthogonal", 1), ("orthogonal", 3), ("perspective", 2)])
def test_exact_nodes_scatter(emu, tmp_path, proj, sms):
    c = _case("g_rot", proj)
    outs = _run(tmp_path, "fn", emu["fp32"], [str(sms), "nodes", "17", "9"], c, _points(c, 8))
    assert outs["a"].size == 9 ** 3
    _assert_bits(outs)


# ---- the tensor-core program over a node list and over a grid range ------------------------------------------------------
@pytest.mark.parametrize("src,proj,sms", [("nodes", "orthogonal", 2), ("nodes", "perspective", 3),
                                          ("grid", "orthogonal", 1), ("grid", "perspective", 2)])
def test_tc_nodes_and_grid(emu, tmp_path, src, proj, sms):
    c = _case("g_rot", proj)
    args = [str(sms)] + (["nodes", "17", "5"] if src == "nodes" else ["grid", "9", "3", "2"])
    outs = _run(tmp_path, "t" + src, emu["tc"], args, c, _points(c, 8))
    assert outs["a"].size == (5 ** 3 if src == "nodes" else 2 * 9 * 9)
    _assert_bits(outs)


# ---- the colour surface render of both programs ----------------------------------------------------------------------------
def _vertex_rows(n=120, seed=7):
    g = torch.Generator().manual_seed(seed)
    cols = torch.randperm(R * R, generator=g)[:n]
    return torch.stack([(cols // R).float(), (cols % R).float(), torch.rand(n, generator=g) * (R - 1)]).numpy()


@pytest.mark.parametrize("program,proj,sms", [("fp32", "orthogonal", 3), ("fp32", "perspective", 1),
                                              ("tc", "orthogonal", 2), ("tc", "perspective", 3)])
def test_colour_surface(emu, tmp_path, program, proj, sms):
    c = _case("c_rot", proj)
    rows = _vertex_rows()
    count = str(rows.shape[1] - 5)                # (the count on the device, below the capacity)
    if program == "fp32":
        outs = _run(tmp_path, "sf", emu["fp32"], [str(sms), "surface", str(R), count] + UNIT, c, rows)
    else:
        outs = _run(tmp_path, "st", emu["tc"], [str(sms), "surface", str(R), count] + UNIT, c, rows)
    assert outs["a"].size == R * R * 3
    _assert_bits(outs)


# ---- the gradient programs -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("proj,sms", [("orthogonal", 1), ("orthogonal", 3), ("perspective", 2)])
def test_exact_gradient(emu, tmp_path, proj, sms):
    c = _case("g_rot", proj)
    outs = _run(tmp_path, "g", emu["fp32"], [str(sms), "grad"], c, _points(c, 37))
    _assert_bits(outs, min_distinct=37)


@pytest.mark.parametrize("proj,sms", [("orthogonal", 2), ("perspective", 1), ("perspective", 3)])
def test_tc_gradient(emu, tmp_path, proj, sms):
    c = _case("g_rot", proj)
    outs = _run(tmp_path, "j", emu["tc"], [str(sms), "jvp"], c, _points(c, 35))
    _assert_bits(outs, min_distinct=35)
    # the gradient rows (after the value row) differ too: the Jacobian reads the buffer as well
    a, b = outs["a"][35:], outs["b"][35:]
    assert int((a.view(np.uint32) != b.view(np.uint32)).sum()) >= 35

