"""CPU checks of the point gradient of query() (mp_query_points_grad): the differentiable restatement against the reference's
autograd goldens, and the gradient kernel -- compiled unmodified on the CPU model of tests/emu -- against those goldens, against
the fp32 query kernel's values bit for bit, across simulated SM counts, outside the image, and under the range guard and a
device-side point count."""
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import spec
from emu_harness import build, write_input
from grad_cases import grad_cases, load_grad_case, query_grad_ref, within_bar


def test_grad_goldens_cover_the_cases():
    assert set(grad_cases()) >= {"g_rot", "g_persp", "g_nocalib", "g_bigfeat", "c_rot"}
    assert load_grad_case("c_rot")["grad_output"] is not None


@pytest.mark.parametrize("name", grad_cases())
def test_restatement_matches_reference_grad_golden(name):
    c = load_grad_case(name)
    _, g64 = query_grad_ref(c["feat"], c["points"], c["calib"], c["Ws"], c["bs"], c["last_op"], c["proj"],
                            grad_output=c["grad_output"], dtype=torch.float64)
    assert (g64 - c["grad64"]).abs().max().item() <= 1e-9 * c["grad64"].abs().max().item()
    val, g32 = query_grad_ref(c["feat"], c["points"], c["calib"], c["Ws"], c["bs"], c["last_op"], c["proj"],
                            grad_output=c["grad_output"])
    assert (val - c["value"]).abs().max().item() < 2e-6
    ok, msg = within_bar(g32, c["grad32"])
    assert ok, msg


# ---- the kernel on the CPU model -------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    """(gradient harness, fp32 query harness)"""
    return build(tmp_path_factory, "emu_query_grad"), build(tmp_path_factory, "emu_query_fp32")


def _write_input(path, c, n):
    write_input(path, c["feat"], c["points"][:, :, :n], c["calib"], c["proj"], c["chans"][-1], c["last_op"], c["Ws"], c["bs"])


def _run_grad(emu, tmp_path, c, n, sms=3, tag="g", env=None):
    """-> (value [Res,n], dpoints [3,n]) of the gradient kernel"""
    res = c["chans"][-1]
    fin, fout = str(tmp_path / ("in_%s.bin" % tag)), str(tmp_path / ("out_%s.f32" % tag))
    _write_input(fin, c, n)
    args = [emu[0], fin, fout, str(sms)]
    if c["grad_output"] is not None:
        fg = str(tmp_path / ("gout_%s.f32" % tag))
        c["grad_output"][:, :n].contiguous().numpy().astype(np.float32).tofile(fg)
        args.append(fg)
    r = subprocess.run(args, capture_output=True, text=True, timeout=1800, env=dict(os.environ, **(env or {})))
    assert r.returncode == 0, r.stderr[-2000:]
    out = torch.from_numpy(np.fromfile(fout, dtype=np.float32))
    assert out.numel() == (res + 3) * n
    return out[:res * n].reshape(res, n), out[res * n:].reshape(3, n)


def _run_fp32(emu, tmp_path, c, n):
    fin, fout = str(tmp_path / "in_q.bin"), str(tmp_path / "out_q.f32")
    _write_input(fin, c, n)
    r = subprocess.run([emu[1], fin, fout], capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-2000:]
    return torch.from_numpy(np.fromfile(fout, dtype=np.float32)).reshape(c["chans"][-1], n)


# the first 8 points of every case are border_points(): on the image border / corners and far outside
@pytest.mark.parametrize("name,n", [("g_rot", 40), ("g_persp", 37), ("g_nocalib", 35), ("g_bigfeat", 33), ("c_rot", 34)])
def test_kernel_matches_reference_grad_golden(emu, tmp_path, name, n):
    c = load_grad_case(name)
    val, dp = _run_grad(emu, tmp_path, c, n)
    assert (val - c["value"][:, :n]).abs().max().item() <= 2e-5
    ok, msg = within_bar(dp, c["grad32"][:, :n])
    assert ok, msg


@pytest.mark.parametrize("name", ["g_rot", "c_rot"])
def test_kernel_value_is_the_fp32_query_bit_for_bit(emu, tmp_path, name):
    c = load_grad_case(name)
    n = 35
    val, _ = _run_grad(emu, tmp_path, c, n)
    assert torch.equal(val, _run_fp32(emu, tmp_path, c, n))


def test_kernel_is_identical_on_1_to_3_sms(emu, tmp_path):
    c = load_grad_case("g_nocalib")
    n = 50                    # 4 tiles of 16 points, the last one ragged
    want = _run_grad(emu, tmp_path, c, n, sms=1, tag="s1")
    for sms in (2, 3):
        got = _run_grad(emu, tmp_path, c, n, sms=sms, tag="s%d" % sms)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]), sms


def test_kernel_gradient_is_exactly_zero_outside_the_image(emu, tmp_path):
    c = load_grad_case("g_rot")
    n = 48
    _, dp = _run_grad(emu, tmp_path, c, n)
    xyz = spec.project_ref(c["points"][0, :, :n], c["calib"][0])
    outside = ~((xyz[0] >= -1) & (xyz[0] <= 1) & (xyz[1] >= -1) & (xyz[1] <= 1))
    assert int(outside.sum()) >= 3
    assert bool((dp[:, outside] == 0).all())
    assert bool((dp[:, ~outside].abs().sum(0) > 0).all())


def test_kernel_range_guard_and_device_count(emu, tmp_path):
    """One map above the head's feature limit and one below: a launch guarded out of range writes the value and d points
    only for the map above, one guarded in range only for the map below.  The device-side count stops the launch at that
    point."""
    c = load_grad_case("g_rot")
    n = 40
    full = _run_grad(emu, tmp_path, c, n)
    for guard, runs_above in (("2", True), ("1", False)):
        for amax, above in (("2", True), ("0.5", False)):
            got = _run_grad(emu, tmp_path, c, n, tag="g%s%s" % (guard, amax),
                            env={"EMU_GUARD": guard, "EMU_TC_LIMIT": "1", "EMU_AMAX": amax})
            if above == runs_above:
                assert torch.equal(got[0], full[0]) and torch.equal(got[1], full[1]), (guard, amax)
            else:
                assert bool((got[0] == -4242).all()) and bool((got[1] == -4242).all()), (guard, amax)
    k = 21
    cut = _run_grad(emu, tmp_path, c, n, tag="cnt", env={"EMU_COUNT": str(k)})
    assert torch.equal(cut[0][:, :k], full[0][:, :k]) and torch.equal(cut[1][:, :k], full[1][:, :k])
    assert bool((cut[0][:, k:] == -4242).all()) and bool((cut[1][:, k:] == -4242).all())
