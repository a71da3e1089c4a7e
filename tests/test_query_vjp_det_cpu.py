"""CPU checks of the ordered feature gradient of the training query (mp_query_points_vjp_ex with MP_VJP_DETERMINISTIC): the VJP
kernel, the radix sort and the gather of query_vjp.cu compiled unmodified on the CPU model of tests/emu.  d features against
the reference's goldens and the atomic path, the same bits at every SM count and for every request, the other gradients
the flag-off bits, crowded cells and the map's edges, a restatement of the documented order from a dump of the scratch
(the --dump option of tests/emu/emu_fp32.cpp's vjp op), and the ptxas report of the new kernels."""
import re

import pytest
import torch

from emu_harness import build, ptxas_report
from ordered_cases import one_cell_case, read_dump, restate_ordered_dfeat
from vjp_cases import flat, golden_bar, load_vjp_case, query_vjp_ref, rel_dist, run_vjp, vjp_bar

DET = 1                                     # MP_VJP_DETERMINISTIC


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return build(tmp_path_factory, "emu_fp32")


def _run(emu, tmp_path, c, flags, chunk=0, sms=3, want="fpw", tag="v", dump=None):
    """stage 0 of a case on the CPU model -> (dfeat [B,C,H,W], dpoints [B,3,N], [dW_l], [db_l])"""
    gout = "-" if c["grad_output"] is None else c["grad_output"][0].contiguous()
    return run_vjp(emu, tmp_path, c, c["feats"][0], gout, chunk, want, options=dict(sms=sms, vjp_flags=flags, dump=dump),
                   tag=tag)[:4]


def _close_to_atomic(det, atomic):
    return (det - atomic).abs().max().item() <= 1e-6 * atomic.abs().max().item()


# every single-stage golden; 64-point chunks, so that several chunks add into the map
@pytest.mark.parametrize("name", ["g_b1_rot", "g_b1_nocalib_nonsquare", "c_b3_rot"])
def test_ordered_feature_gradient_matches_reference_golden(emu, tmp_path, name):
    c = load_vjp_case(name)
    assert len(c["feats"]) == 1
    det = _run(emu, tmp_path, c, DET, chunk=64, tag="det")
    ok, msg = golden_bar(flat(det[0]), c, "dfeat")
    assert ok, msg
    # the other three gradients are the flag-off bits; d features the atomic sums up to their order
    off = _run(emu, tmp_path, c, 0, chunk=64, tag="off")
    assert torch.equal(det[1], off[1])
    for x, y in zip(det[2] + det[3], off[2] + off[3]):
        assert torch.equal(x, y)
    assert _close_to_atomic(det[0], off[0])


def test_ordered_feature_gradient_is_the_same_bits_at_every_sm_count_and_request(emu, tmp_path):
    c = load_vjp_case("narrow_b3_persp")
    runs = [_run(emu, tmp_path, c, DET, chunk=48, sms=s, tag="s%d" % s) for s in (1, 2, 3)]
    for r in runs[1:]:
        assert torch.equal(r[0], runs[0][0])
        assert torch.equal(r[1], runs[0][1])
    only_f = _run(emu, tmp_path, c, DET, chunk=48, sms=2, want="f", tag="f")
    assert torch.equal(only_f[0], runs[0][0])
    assert bool((only_f[1] == 0).all()) and all(bool((w == 0).all()) for w in only_f[2] + only_f[3])
    off = _run(emu, tmp_path, c, 0, chunk=48, tag="off")
    assert torch.equal(runs[0][1], off[1])
    for x, y in zip(runs[0][2] + runs[0][3], off[2] + off[3]):
        assert torch.equal(x, y)
    assert _close_to_atomic(runs[0][0], off[0])
    r = query_vjp_ref(c["feats"][:1], c["points"], c["calib"], c["Ws"], c["bs"], c["last_op"], c["proj"],
                      None if c["grad_output"] is None else c["grad_output"][:1])
    assert (flat(runs[0][0]) - flat(r["dfeat"])).abs().max().item() <= 1e-4 * flat(r["dfeat"]).abs().max().item()


def test_crowded_cell_edges_and_outside_points(emu, tmp_path):
    """two images of 300 points, all but 8 of each in one cell; the 8 on the last row and column, the far corners and
    outside the image.  Several chunks, one chunk, the atomic path and the float64 restatement."""
    c = one_cell_case(2, 300, 16, 16)
    args = (c["feats"], c["points"], c["calib"], c["Ws"], c["bs"], c["last_op"], c["proj"], c["grad_output"])
    r64, r32 = query_vjp_ref(*args, dtype=torch.float64), query_vjp_ref(*args, dtype=torch.float32)
    dump = str(tmp_path / "dump.bin")
    one = _run(emu, tmp_path, c, DET, chunk=0, want="f", tag="one", dump=dump)
    many = _run(emu, tmp_path, c, DET, chunk=40, want="f", tag="many")
    atomic = _run(emu, tmp_path, c, 0, chunk=0, want="f", tag="atomic")
    for got in (one[0], many[0]):
        ok, msg = vjp_bar(got, r64["dfeat"][0], rel_dist(r32["dfeat"][0], r64["dfeat"][0]))
        assert ok, msg
    # (one chunk: the atomic path's terms in another order; 40-point chunks also add partial sums of the crowded cell)
    assert _close_to_atomic(one[0], atomic[0])
    # the texels of the crowded cells and the edge points' taps hold gradient, the rest of the map none
    touched = r64["dfeat"][0].abs().sum(1) > 0
    assert torch.equal(one[0].abs().sum(1) > 0, touched)
    assert bool(touched[:, -1, :].any()) and bool(touched[:, :, -1].any())
    want = restate_ordered_dfeat(*read_dump(dump), 2, 16, 16)
    assert torch.equal(one[0], want)


def test_dump_restates_the_documented_order_on_a_golden(emu, tmp_path):
    c = load_vjp_case("g_b1_rot")
    dump = str(tmp_path / "dump.bin")
    dfeat = _run(emu, tmp_path, c, DET, chunk=0, want="fw", tag="dump", dump=dump)[0]
    B, C, H, W = c["feats"][0].shape
    want = restate_ordered_dfeat(*read_dump(dump), B, H, W)
    assert torch.equal(dfeat, want)


# ---- ptxas report ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kernel,count", [("radix_count_kernel", 1), ("radix_scatter_kernel", 1), ("dfeat_gather_kernel", 1),
                                          ("DigitCounts", 2)])
def test_ordered_path_kernels_have_no_spill_and_no_stack_frame(kernel, count):
    found = {name: " ".join(lines) for name, lines in ptxas_report("query_vjp.cu")[0] if kernel in name}
    assert len(found) == count, list(found)
    for name, stats in found.items():
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", stats)
        assert m and m.groups() == ("0", "0", "0"), (name, stats)
