"""CPU checks of the differentiable query for training (mp_query_points_vjp): the float64 restatement against the reference's
train-mode autograd goldens, and the VJP kernel with its weight-gradient contraction -- compiled unmodified on the CPU model of
tests/emu -- against those goldens, its point gradient against the gradient kernel's bit for bit, its determinism across chunk
sizes and SM counts.  Also the ptxas report: no spill and no stack frame for the new kernels, and the register counts of the
query and gradient kernels."""
import re
import subprocess

import numpy as np
import pytest
import torch

import emu_harness
from emu_harness import build, ptxas_report, write_input
from vjp_cases import GRAD_NAMES, flat, golden_bar, load_vjp_case, query_vjp_ref, vjp_cases

emu_harness.HARNESSES.setdefault("emu_query_vjp", ("-O3", True))


def test_vjp_goldens_cover_the_cases():
    names = set(vjp_cases())
    assert len(names) >= 6
    cs = [load_vjp_case(n) for n in names]
    assert {len(c["feats"]) for c in cs} >= {1, 4} and {c["points"].shape[0] for c in cs} >= {1, 3}
    assert {c["proj"] for c in cs} == {"orthogonal", "perspective"} and any(c["calib"] is None for c in cs)
    assert any(c["feats"][0].shape[2] != c["feats"][0].shape[3] for c in cs)
    assert any(c["grad_output"] is not None for c in cs) and {c["chans"][-1] for c in cs} >= {1, 3}


@pytest.mark.parametrize("name", vjp_cases())
def test_restatement_matches_reference_vjp_golden(name):
    c = load_vjp_case(name)
    r = query_vjp_ref(c["feats"], c["points"], c["calib"], c["Ws"], c["bs"], c["last_op"], c["proj"], c["grad_output"])
    for g in GRAD_NAMES:
        got = flat(r[g])[c["idx_" + g]]
        assert (got - c[g + "64"]).abs().max().item() <= 1e-9 * c["scale_" + g], g
        assert abs(flat(r[g]).abs().max().item() - c["scale_" + g]) <= 1e-9 * c["scale_" + g], g


# ---- the kernels on the CPU model ------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    """(VJP harness, point-gradient harness)"""
    return build(tmp_path_factory, "emu_query_vjp"), build(tmp_path_factory, "emu_query_grad")


def _run_vjp(emu, tmp_path, c, stage=0, chunk=0, sms=3, want="fpw", tag="v"):
    """one stage of a golden on the CPU model -> (dfeat [B,C,H,W], dpoints [B,3,N], [dW_l], [db_l])"""
    feat, pts, chans = c["feats"][stage], c["points"], c["chans"]
    B, C, H, W = feat.shape
    N = pts.shape[2]
    fin, fout = str(tmp_path / ("in_%s.bin" % tag)), str(tmp_path / ("out_%s.f32" % tag))
    write_input(fin, feat, pts, c["calib"], c["proj"], chans[-1], c["last_op"], c["Ws"], c["bs"], batched=True)
    fg = "-"
    if c["grad_output"] is not None:
        fg = str(tmp_path / ("gout_%s.f32" % tag))
        c["grad_output"][stage].contiguous().numpy().astype(np.float32).tofile(fg)
    r = subprocess.run([emu[0], fin, fout, str(B), ",".join(str(x) for x in chans[1:]), fg, str(chunk), str(sms), want],
                       capture_output=True, text=True, timeout=3600)
    assert r.returncode == 0, r.stderr[-2000:]
    out = torch.from_numpy(np.fromfile(fout, dtype=np.float32))
    o = 0

    def take(shape):
        nonlocal o
        k = int(np.prod(shape))
        t = out[o:o + k].reshape(shape)
        o += k
        return t
    dfeat, dp = take((B, C, H, W)), take((B, 3, N))
    dW = [take((chans[l + 1], c["Ws"][l].shape[1])) for l in range(len(c["Ws"]))]
    db = [take((chans[l + 1],)) for l in range(len(c["Ws"]))]
    assert o == out.numel()
    return dfeat, dp, dW, db


# the single-stage goldens (a multi-stage golden's head gradient sums over its stages: the restatement covers those)
SINGLE = ["g_b1_rot", "g_b1_nocalib_nonsquare", "c_b3_rot"]


@pytest.mark.parametrize("name", SINGLE)
def test_kernel_matches_reference_vjp_golden(emu, tmp_path, name):
    c = load_vjp_case(name)
    assert len(c["feats"]) == 1
    dfeat, dp, dW, db = _run_vjp(emu, tmp_path, c)
    for g, got in (("dfeat", dfeat), ("dpoints", dp), ("dW", dW), ("db", db)):
        ok, msg = golden_bar(flat(got), c, g)
        assert ok, msg


def test_kernel_matches_restatement_on_every_stage_of_a_multistage_golden(emu, tmp_path):
    c = load_vjp_case("narrow_b3_persp")
    dW_sum = None
    for s in range(len(c["feats"])):
        dfeat, dp, dW, db = _run_vjp(emu, tmp_path, c, stage=s, tag="s%d" % s)
        r = query_vjp_ref([c["feats"][s]], c["points"], c["calib"], c["Ws"], c["bs"], c["last_op"], c["proj"],
                          None if c["grad_output"] is None else [c["grad_output"][s]])
        for g, got in (("dfeat", [dfeat]), ("dW", dW), ("db", db)):
            ref = flat(r[g])
            assert (flat(got) - ref).abs().max().item() <= 1e-4 * ref.abs().max().item(), (s, g)
        dW_sum = flat(dW) if dW_sum is None else dW_sum + flat(dW)
    ok, msg = golden_bar(dW_sum, c, "dW")
    assert ok, msg


def test_kernel_point_gradient_is_the_gradient_kernels_bit_for_bit(emu, tmp_path):
    c = load_vjp_case("g_b1_rot")
    _, dp, _, _ = _run_vjp(emu, tmp_path, c, want="p")
    fin, fout = str(tmp_path / "in_g.bin"), str(tmp_path / "out_g.f32")
    write_input(fin, c["feats"][0], c["points"][0], c["calib"], c["proj"], 1, c["last_op"], c["Ws"], c["bs"])
    r = subprocess.run([emu[1], fin, fout, "3"], capture_output=True, text=True, timeout=3600)
    assert r.returncode == 0, r.stderr[-2000:]
    N = c["points"].shape[2]
    want = torch.from_numpy(np.fromfile(fout, dtype=np.float32))[N:].reshape(3, N)
    assert torch.equal(dp[0], want)


def test_kernel_gradients_are_deterministic_and_requests_independent(emu, tmp_path):
    c = load_vjp_case("c_b3_rot")
    a = _run_vjp(emu, tmp_path, c, chunk=48, sms=2, tag="a")
    b = _run_vjp(emu, tmp_path, c, chunk=48, sms=3, tag="b")
    assert torch.equal(a[1], b[1])
    for x, y in zip(a[2] + a[3], b[2] + b[3]):
        assert torch.equal(x, y)
    # only the weights: the same bits; only the features: the same up to the atomics' order
    w = _run_vjp(emu, tmp_path, c, chunk=48, want="w", tag="w")
    for x, y in zip(a[2] + a[3], w[2] + w[3]):
        assert torch.equal(x, y)
    assert bool((w[0] == 0).all()) and bool((w[1] == 0).all())
    f = _run_vjp(emu, tmp_path, c, want="f", tag="f")
    assert (f[0] - a[0]).abs().max().item() <= 1e-6 * a[0].abs().max().item()
    # one chunk: another summation order of the same sums
    one = _run_vjp(emu, tmp_path, c, chunk=0, want="w", tag="one")
    ok, msg = golden_bar(flat(one[2]), c, "dW")
    assert ok, msg


# ---- ptxas report ----------------------------------------------------------------------------------------------------------
def _stats(source, kernel):
    return {name: " ".join(lines) for name, lines in ptxas_report(source)[0] if kernel in name}


@pytest.mark.parametrize("source,kernel,count", [("query_fp32.cu", "query_vjp_kernel", 3), ("query_vjp.cu", "wgrad_kernel", 1),
                                                 ("query_vjp.cu", "nhwc_to_nchw_kernel", 1)])
def test_new_kernels_have_no_spill_and_no_stack_frame(source, kernel, count):
    found = _stats(source, kernel)
    assert len(found) == count, list(found)
    for name, stats in found.items():
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", stats)
        assert m and m.groups() == ("0", "0", "0"), (name, stats)


# registers of the query and gradient kernels (P, SURF) as they were before the VJP kernel joined their source file
REGISTERS = {("query_grad_kernel", "8"): 103, ("query_grad_kernel", "16"): 119, ("query_grad_kernel", "32"): 157,
             ("query_fp32_kernel", "8ELb1"): 102, ("query_fp32_kernel", "16ELb1"): 118, ("query_fp32_kernel", "32ELb1"): 145,
             ("query_fp32_kernel", "8ELb0"): 102, ("query_fp32_kernel", "16ELb0"): 125, ("query_fp32_kernel", "32ELb0"): 145}


def test_query_and_gradient_kernels_keep_their_registers():
    entries = ptxas_report("query_fp32.cu")[0]
    for (kernel, tag), regs in REGISTERS.items():
        hits = [" ".join(lines) for name, lines in entries if "%sILi%s" % (kernel, tag) in name]
        assert len(hits) == 1, (kernel, tag)
        m = re.search(r"Used (\d+) registers", hits[0])
        assert m and int(m.group(1)) == regs, (kernel, tag, hits[0])
