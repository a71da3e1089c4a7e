"""CPU checks of the training query's backward (mp_launch_query_vjp) off the goldens' shapes, on the CPU model of tests/emu
(tests/emu/emu_query_vjp_det.cpp: query_vjp_kernel, wgrad_kernel, the radix sort, the gather and the layout step compiled
unmodified): the ordered feature gradient at one, two and three radix passes and with several radix blocks, an image of a
batch against the same image alone where the two take different pass counts, per-layer partial weight / bias requests, and
hidden units whose pre-activation is exactly 0."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import emu_harness
from emu_harness import build, write_input
from ordered_cases import GPU_RADIX_CASES, radix_passes_rule, read_dump, restate_ordered_dfeat, spread_case, zero_unit_case
from vjp_cases import query_vjp_ref, rel_dist, vjp_bar

emu_harness.HARNESSES.setdefault("emu_query_vjp_det", ("-O3", True))

DET = 1                                     # MP_VJP_DETERMINISTIC


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return build(tmp_path_factory, "emu_query_vjp_det")


def _run(emu, tmp_path, c, flags, chunk=0, sms=3, want="fpw", tag="v", env=None):
    """stage 0 of a case on the CPU model -> (dfeat [B,C,H,W], dpoints [B,3,N], [dW_l], [db_l], stdout)"""
    feat, pts, chans = c["feats"][0], c["points"], c["chans"]
    B, C, H, W = feat.shape
    N = pts.shape[2]
    fin, fout = str(tmp_path / ("in_%s.bin" % tag)), str(tmp_path / ("out_%s.f32" % tag))
    write_input(fin, feat, pts, c["calib"], c["proj"], chans[-1], c["last_op"], c["Ws"], c["bs"], batched=True)
    fg = str(tmp_path / ("gout_%s.f32" % tag))
    c["grad_output"][0].contiguous().numpy().astype(np.float32).tofile(fg)
    r = subprocess.run([emu, fin, fout, str(B), ",".join(str(x) for x in chans[1:]), fg, str(chunk), str(sms), want],
                       capture_output=True, text=True, timeout=3600, env=dict(os.environ, EMU_VJP_FLAGS=str(flags), **(env or {})))
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
    dW = [take(tuple(w.shape)) for w in c["Ws"]]
    db = [take(tuple(b.shape)) for b in c["bs"]]
    assert o == out.numel()
    return dfeat, dp, dW, db, r.stdout


def _ref(c, dtype):
    return query_vjp_ref(c["feats"], c["points"], c["calib"], c["Ws"], c["bs"], c["last_op"], c["proj"], c["grad_output"],
                         dtype=dtype)


# ---- every radix-pass count ------------------------------------------------------------------------------------------------
# (B, H, W, N per image, bands of the last image, the passes): one chunk of more than 2048 columns, several radix blocks
RADIX = {
    "one_pass": (1, 12, 16, 2080, (), 1),
    "two_passes": (2, 40, 40, 1040, (), 2),
    "three_passes": (1, 256, 260, 2080, ((253, 256), (240, 253)), 3),
}


def test_radix_cases_take_every_pass_count():
    """the rule of radix_passes restated: this file's cases and the GPU's together take 1, 2, 3 and 4 passes"""
    assert [radix_passes_rule(n) for n in (1, 255, 256, 65535, 65536, (1 << 24) - 1, 1 << 24, 0xFFFFFFFE)] == \
        [1, 1, 2, 2, 3, 3, 4, 4]
    seen = set()
    for B, H, W, N, _, passes in RADIX.values():
        assert radix_passes_rule(B * H * W) == passes
        seen.add(passes)
    assert radix_passes_rule(3 * 10 * 10) == 2 and radix_passes_rule(10 * 10) == 1          # the batch against one image
    for B, H, W, _, _ in GPU_RADIX_CASES.values():
        assert radix_passes_rule(B * H * W) == radix_passes_rule(H * W) + 1
        seen |= {radix_passes_rule(B * H * W), radix_passes_rule(H * W)}
    assert seen == {1, 2, 3, 4}


@pytest.mark.parametrize("name", sorted(RADIX))
def test_ordered_feature_gradient_at_every_radix_pass_count(emu, tmp_path, name):
    B, H, W, N, bands, passes = RADIX[name]
    c = spread_case(B, N, H, W, bands=bands, seed=len(name))
    dump = str(tmp_path / "dump.bin")
    det = _run(emu, tmp_path, c, DET, want="f", tag="det", env=dict(EMU_VJP_DUMP=dump))
    assert re.search(r"radix passes (\d)", det[4]).group(1) == str(passes)
    dx, wgt, keys, order = read_dump(dump)
    assert len(keys) > 2048                                    # several radix blocks
    if bands:
        assert int(keys[keys < B * H * W].max()) >= 1 << 16    # keys that the third pass sorts
    assert torch.equal(det[0], restate_ordered_dfeat(dx, wgt, keys, order, B, H, W))
    r64, r32 = _ref(c, torch.float64), _ref(c, torch.float32)
    ok, msg = vjp_bar(det[0], r64["dfeat"][0], rel_dist(r32["dfeat"][0], r64["dfeat"][0]))
    assert ok, msg
    atomic = _run(emu, tmp_path, c, 0, want="f", tag="atomic")[0]
    assert (det[0] - atomic).abs().max().item() <= 1e-6 * atomic.abs().max().item()


def test_an_image_of_a_batch_is_that_image_alone_at_another_pass_count(emu, tmp_path):
    """one chunk: B = 3 maps of 10 x 10 take 2 passes, one of them alone 1; image b's columns keep their order"""
    c = spread_case(3, 150, 10, 10, seed=7)
    batch = _run(emu, tmp_path, c, DET, want="f", tag="batch", env=dict(EMU_VJP_DUMP=str(tmp_path / "b.bin")))
    assert "radix passes 2" in batch[4]
    for b in range(3):
        cb = dict(c, feats=[c["feats"][0][b:b + 1]], points=c["points"][b:b + 1], grad_output=[c["grad_output"][0][b:b + 1]])
        alone = _run(emu, tmp_path, cb, DET, want="f", tag="a%d" % b, env=dict(EMU_VJP_DUMP=str(tmp_path / "a.bin")))
        assert "radix passes 1" in alone[4]
        assert torch.equal(batch[0][b:b + 1], alone[0]), b


# ---- per-layer partial requests --------------------------------------------------------------------------------------------
FULL = 0xFF
# (d W mask, d b mask) over the 8 layers of the deep head: null d W for some layers, null d b for others, one layer entirely
# null, the first, the last, and only two middle layers
PARTIAL = [(0b10100101, FULL), (FULL, 0b01011010), (FULL & ~(1 << 3), FULL & ~(1 << 3)), (FULL & ~1, FULL & ~1),
           (FULL & ~(1 << 7), FULL & ~(1 << 7)), (0b00000100, 0b00100000)]


@pytest.mark.parametrize("flags", [0, DET])
def test_partial_requests_write_exactly_the_requested_layers(emu, tmp_path, flags):
    """every array passed is the full request's bits; every one left null keeps the sentinel (-7)"""
    c = spread_case(2, 90, 12, 5, chans=[40, 32, 32, 33, 31, 64, 16, 8, 1], seed=11)
    full = _run(emu, tmp_path, c, flags, chunk=64, tag="full")
    assert all(bool((t != 0).any()) for t in full[2] + full[3])
    for i, (wm, bm) in enumerate(PARTIAL):
        got = _run(emu, tmp_path, c, flags, chunk=64, tag="p%d" % i, env=dict(EMU_VJP_WMASK=str(wm), EMU_VJP_BMASK=str(bm)))
        assert torch.equal(got[1], full[1])
        for l in range(8):
            for mask, g, f in ((wm, got[2][l], full[2][l]), (bm, got[3][l], full[3][l])):
                if (mask >> l) & 1:
                    assert torch.equal(g, f), (i, l)
                else:
                    assert bool((g == -7.0).all()), (i, l)


# ---- pre-activations of exactly 0 ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("flags", [0, DET])
def test_pre_activations_of_exactly_zero_take_the_slope_at_zero(emu, tmp_path, flags):
    """lrelu' at 0 is the negative slope (torch's leaky_relu backward): every gradient within its bar of the float64
    restatement, and the rows of the zero units within the bar of their own scale"""
    c, zero_rows = zero_unit_case()
    got = _run(emu, tmp_path, c, flags, chunk=96)
    r64, r32 = _ref(c, torch.float64), _ref(c, torch.float32)
    for i, g in enumerate(("dfeat", "dpoints", "dW", "db")):
        mine = [got[0]] if g == "dfeat" else got[i]
        ok, msg = vjp_bar(mine, r64[g], rel_dist(r32[g], r64[g]))
        assert ok, (g, msg)
    for l, rows in zero_rows.items():
        for g, i in (("dW", 2), ("db", 3)):
            ref = r64[g][l][rows]
            assert ref.abs().max().item() > 0
            ok, msg = vjp_bar(got[i][l][rows], ref, rel_dist(r32[g][l][rows], ref))
            assert ok, (l, g, msg)
    # the units that see only the depth: the points with z = 0 carry their d z through the slope at 0
    z0 = c["points"][:, 2] == 0
    ref = r64["dpoints"][:, 2][z0]
    ok, msg = vjp_bar(got[1][:, 2][z0], ref, rel_dist(r32["dpoints"][:, 2][z0], ref))
    assert ok, msg
