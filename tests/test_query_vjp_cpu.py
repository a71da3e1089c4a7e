"""CPU checks of the differentiable query for training (mp_query_points_vjp): the float64 restatement against the reference's
train-mode autograd goldens, and the VJP kernel with its weight-gradient contraction -- compiled unmodified on the CPU model of
tests/emu -- against those goldens, its point gradient against the single-map gradient launch's bit for bit, its determinism
across chunk sizes and SM counts.  Also the ptxas report: no spill and no stack frame for the new kernels, and the register
counts of the query kernel."""
import re

import pytest
import torch

from oracle import spec
from emu_harness import build, ptxas_report, run
from head_cases import fp32_tile
from vjp_cases import GRAD_NAMES, flat, golden_bar, load_vjp_case, query_vjp_ref, run_vjp, vjp_cases


def test_vjp_goldens_cover_the_cases():
    names = set(vjp_cases())
    assert len(names) >= 6
    cs = [load_vjp_case(n) for n in names]
    assert {len(c["feats"]) for c in cs} >= {1, 4} and {c["points"].shape[0] for c in cs} >= {1, 3}
    assert {c["proj"] for c in cs} == {"orthogonal", "perspective"} and any(c["calib"] is None for c in cs)
    assert any(c["feats"][0].shape[2] != c["feats"][0].shape[3] for c in cs)
    assert any(c["grad_output"] is not None for c in cs) and {c["chans"][-1] for c in cs} >= {1, 3}
    # the reverse tiles 8, 16 and 32, each exactly full once: one more unit in the second hidden layer takes another tile
    chans = [c["chans"] for c in cs]
    tiles = {fp32_tile(ch, grad=True) for ch in chans}
    assert tiles >= {8, 16, 32}, tiles
    for P in (8, 16, 32):
        assert any(fp32_tile(ch, grad=True) == P and fp32_tile(ch[:2] + [ch[2] + 1] + ch[3:], grad=True) != P
                   for ch in chans if len(ch) >= 4), P
    # one layer and MP_MAX_LAYERS; wgrad_kernel's bias column alone in the last k-tile and last in a full one; outputs of
    # 64 and 65 channels; a map of fewer than 32 channels; no last op
    assert {len(ch) - 1 for ch in chans} >= {1, 8}
    cins = {ch[l] + (ch[0] if l else 0) for ch in chans for l in range(len(ch) - 1)}
    assert {k % 64 for k in cins} >= {0, 63}, sorted(cins)
    assert {w for ch in chans for w in ch[1:]} >= {64, 65}
    assert any(ch[0] - 1 < 32 for ch in chans)
    assert any(c["last_op"] == spec.LAST_NONE for c in cs)
    # maps one texel high and one wide; B * H * W <= 255, one radix pass of the ordered feature gradient
    shapes = [c["feats"][0].shape for c in cs]
    assert any(s[2] == 1 for s in shapes) and any(s[3] == 1 for s in shapes)
    assert any(s[0] * s[2] * s[3] <= 255 for s in shapes)


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
    return build(tmp_path_factory, "emu_fp32")


def _run_vjp(emu, tmp_path, c, stage=0, chunk=0, sms=3, want="fpw", tag="v"):
    """one stage of a golden on the CPU model -> (dfeat [B,C,H,W], dpoints [B,3,N], [dW_l], [db_l])"""
    gout = "-" if c["grad_output"] is None else c["grad_output"][stage].contiguous()
    return run_vjp(emu, tmp_path, c, c["feats"][stage], gout, chunk, want, options=dict(sms=sms), tag=tag)[:4]


# the single-stage goldens (a multi-stage golden's head gradient sums over its stages: the restatement covers those)
SINGLE = ["g_b1_rot", "g_b1_nocalib_nonsquare", "c_b3_rot", "p8_b2_persp", "odd_b2_persp", "tiles_b1_rot", "single_b2_nocalib",
          "deep_b1_rot", "row_b1_rot", "col_b2_nocalib", "tiny_b3"]


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
    """the batched launcher's d points against mp_launch_query_grad's: one map, guarded (out of range, so it runs) and with
    the point count on the device"""
    c = load_vjp_case("g_b1_rot")
    _, dp, _, _ = _run_vjp(emu, tmp_path, c, want="p")
    N = c["points"].shape[2]
    inp = dict(feat=c["feats"][0], rows=c["points"][0], calib=c["calib"], proj=c["proj"], res=1, last_op=c["last_op"],
               Ws=c["Ws"], bs=c["bs"])
    out, _ = run(emu, tmp_path, "grad", inp=inp, shape=(4 * N,), options=dict(sms=3, guard="out", limit=1, amax=2, count=N),
                 tag="g")
    want = out[N:].reshape(3, N)
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


# registers of the query kernel (P, SURF) as they were before the VJP kernel joined its source file
REGISTERS = {("query_fp32_kernel", "8ELb1"): 102, ("query_fp32_kernel", "16ELb1"): 118, ("query_fp32_kernel", "32ELb1"): 145,
             ("query_fp32_kernel", "8ELb0"): 102, ("query_fp32_kernel", "16ELb0"): 125, ("query_fp32_kernel", "32ELb0"): 145}


def test_query_kernel_keeps_its_registers():
    entries = ptxas_report("query_fp32.cu")[0]
    for (kernel, tag), regs in REGISTERS.items():
        hits = [" ".join(lines) for name, lines in entries if "%sILi%s" % (kernel, tag) in name]
        assert len(hits) == 1, (kernel, tag)
        m = re.search(r"Used (\d+) registers", hits[0])
        assert m and int(m.group(1)) == regs, (kernel, tag, hits[0])
