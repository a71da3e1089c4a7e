"""CPU tier of the per-frame camera: every program a captured frame launches, compiled unmodified against the CPU emulation
layer (tests/emu), reads its camera from device memory (a single-map MpBatch whose calibs point at a 12-float buffer, the
--dcal option of tests/emu/emu_fp32.cpp and emu_tc.cpp) and must give, bit for bit, what its by-value launch gives with the
same 12 floats -- the exact query over a node list with the volume scatter, the tensor-core query over a node list and over
a grid range, the colour surface render of both programs, and both gradient programs.  Every case runs two launches
through one buffer rewritten between them, and each must give its own camera's result."""
import numpy as np
import pytest
import torch

from oracle import spec
from emu_harness import build, needs_emu, run
from grad_cases import load_grad_case

pytestmark = needs_emu

R = 65
UNIT = ["-1", "-1", "-1", "1", "1", "1"]


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return {k: build(tmp_path_factory, "emu_" + k) for k in ("fp32", "tc")}


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


def _run(tmp_path, tag, exe, args, c, rows, sms, size):
    """the by-value launches with camera A (the case's) and camera B, and the device-calib pair (B, then A) through one
    buffer (--dcal) -> the four outputs as raw float32 arrays of `size` floats"""
    cal_b = _second_camera(c)
    outs = {}
    for key, calib, dcal in (("a", c["calib"], None), ("b", cal_b, None), ("d", c["calib"], cal_b[0, :3, :4].reshape(-1))):
        inp = dict(feat=c["feat"], rows=rows, calib=calib, proj=c["proj"], res=c["chans"][-1], last_op=c["last_op"],
                   Ws=c["Ws"], bs=c["bs"])
        out, _ = run(exe, tmp_path, *args, inp=inp, shape=(size,), options=dict(sms=sms, dcal=dcal), tag=tag + key)
        outs[key] = out.numpy()
    outs["d_first"] = np.fromfile(str(tmp_path / ("out_%sd.f32.first" % tag)), dtype=np.float32)   # (run's out.f32 + .first)
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
    outs = _run(tmp_path, "fn", emu["fp32"], ["nodes", 17, 9], c, _points(c, 8), sms, 9 ** 3)
    assert outs["a"].size == 9 ** 3
    _assert_bits(outs)


# ---- the tensor-core program over a node list and over a grid range ------------------------------------------------------
@pytest.mark.parametrize("src,proj,sms", [("nodes", "orthogonal", 2), ("nodes", "perspective", 3),
                                          ("grid", "orthogonal", 1), ("grid", "perspective", 2)])
def test_tc_nodes_and_grid(emu, tmp_path, src, proj, sms):
    c = _case("g_rot", proj)
    args, size = (["nodes", 17, 5], 5 ** 3) if src == "nodes" else (["grid", 9, 3, 2], 2 * 9 * 9)
    outs = _run(tmp_path, "t" + src, emu["tc"], args, c, _points(c, 8), sms, size)
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
    count = rows.shape[1] - 5                     # (the count on the device, below the capacity)
    outs = _run(tmp_path, "s" + program[0], emu[program], ["surface", R, count] + UNIT, c, rows, sms, R * R * 3)
    assert outs["a"].size == R * R * 3
    _assert_bits(outs)


# ---- the gradient programs -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("proj,sms", [("orthogonal", 1), ("orthogonal", 3), ("perspective", 2)])
def test_exact_gradient(emu, tmp_path, proj, sms):
    c = _case("g_rot", proj)
    outs = _run(tmp_path, "g", emu["fp32"], ["grad"], c, _points(c, 37), sms, 4 * 37)
    _assert_bits(outs, min_distinct=37)


@pytest.mark.parametrize("proj,sms", [("orthogonal", 2), ("perspective", 1), ("perspective", 3)])
def test_tc_gradient(emu, tmp_path, proj, sms):
    c = _case("g_rot", proj)
    outs = _run(tmp_path, "j", emu["tc"], ["jvp"], c, _points(c, 35), sms, 4 * 35)
    _assert_bits(outs, min_distinct=35)
    # the gradient rows (after the value row) differ too: the Jacobian reads the buffer as well
    a, b = outs["a"][35:], outs["b"][35:]
    assert int((a.view(np.uint32) != b.view(np.uint32)).sum()) >= 35

