"""CPU checks of the batched point gradient (mp_query_points_grad_batch: B images in one launch of each program), with both
gradient programs compiled unmodified on the CPU model of tests/emu -- the tensor-core program's forward-mode derivative
(query_jvp_kernel, `emu_tc_batch jvp --batch B`) and the exact kernel (query_fp32_kernel for the value, query_vjp_kernel
for d points, `emu_fp32_batch grad --batch B`): image b of a batched launch against the single-map launch of image b by
emu_tc / emu_fp32 bit for bit, the range guard per image, the reference's batched autograd goldens
(tests/golden/bgrad_*.npz), and the single-map launch of the tensor-core program against the bytes it gave before it took
a batch."""
import hashlib

import numpy as np
import pytest
import torch

from oracle import spec
import emu_harness
from emu_harness import build, run
from batch_grad_cases import BATCH_GRAD_CASES, load_batch_grad_case, single
from grad_cases import load_grad_case, query_grad_ref, tc_bar, within_bar


# the batched gradient harnesses (tests/emu/emu_tc_batch.cpp, emu_fp32_batch.cpp: emu_tc / emu_fp32 with the batched op),
# built by emu_harness's recipe with the flags of the harnesses they extend
emu_harness.HARNESSES.setdefault("emu_tc_batch", emu_harness.HARNESSES["emu_tc"])
emu_harness.HARNESSES.setdefault("emu_fp32_batch", emu_harness.HARNESSES["emu_fp32"])


@pytest.fixture(scope="module")
def emu_tc(tmp_path_factory):
    """(the single-map harness, the batched one)"""
    return build(tmp_path_factory, "emu_tc"), build(tmp_path_factory, "emu_tc_batch")


@pytest.fixture(scope="module")
def emu_fp32(tmp_path_factory):
    return build(tmp_path_factory, "emu_fp32"), build(tmp_path_factory, "emu_fp32_batch")


def _grad(exes, op, tmp_path, c, n, batched=True, env=None, tag="x", **options):
    """-> (value [B,Res,n], d points [B,3,n]) of `op` ("jvp" on emu_tc, "grad" on emu_fp32) on the first n points of every
    image of c: one batched launch (the batched harness of `exes`), or (batched=False, c holding one image) the single-map
    launch (the single-map harness)"""
    exe = exes[1] if batched else exes[0]
    B, res = c["feat"].shape[0], c["chans"][-1]
    gout = [] if c.get("grad_output") is None else [c["grad_output"][:, :, :n].contiguous()]
    inp = dict(feat=c["feat"], rows=c["points"][:, :, :n], calib=c["calib"], proj=c["proj"], res=res, last_op=c["last_op"],
               Ws=c["Ws"], bs=c["bs"], batched=batched)
    out, _ = run(exe, tmp_path, op, *gout, inp=inp, shape=(B * (res + 3) * n,),
                 options=dict(batch=B if batched else None, **options), env=env, tag=tag)
    return out[:B * res * n].reshape(B, res, n), out[B * res * n:].reshape(B, 3, n)


def _small_colour_case(B=2, H=20, W=24, n=64, seed=601):
    """B colour maps of H x W (non-square), a camera and a seeded grad_output per image: the colour head's program at a size
    the CPU model runs quickly"""
    chans = spec.C_CHANNELS
    Ws, bs = spec.make_weights(chans, seed)
    return dict(net="C", chans=chans, Ws=Ws, bs=bs, last_op=spec.LAST_TANH, proj="orthogonal", B=B,
                feat=torch.cat([spec.make_feat(chans[0] - 1, H, W, seed + 1 + b) for b in range(B)], 0),
                points=torch.cat([spec.make_points(n, seed + 11 + b) for b in range(B)], 0),
                calib=torch.cat([spec.scene_calib(20.0 + 15.0 * b, 33.0 - 40.0 * b) for b in range(B)], 0),
                grad_output=torch.randn(B, chans[-1], n, generator=torch.Generator().manual_seed(seed + 21)))


def _case(name):
    return _small_colour_case() if name == "c_small" else load_batch_grad_case(name)


def _mixed_case():
    """three 32 x 32 geometry maps, the middle one x4 so that exactly it is above the limit of 12"""
    c = load_batch_grad_case("g_nocalib")
    feat = torch.cat([c["feat"][0:1], c["feat"][1:2] * 4.0, c["feat"][0:1] * 0.5], 0)
    pts = torch.cat([c["points"], c["points"][0:1].flip(2)], 0)
    amax = [feat[b].abs().max().item() for b in range(3)]
    assert amax[1] > 12.0 and amax[0] < 12.0 and amax[2] < 12.0, amax
    return dict(c, feat=feat, points=pts, B=3, grad_output=None), amax


def _amax_option(feat):
    """--amax of emu_fp32: each map's largest |feature| (the tensor-core program's G0 kernel finds the same)"""
    return ",".join(repr(float(np.float32(feat[b].abs().max().item()))) for b in range(feat.shape[0]))


def test_batch_grad_goldens_cover_the_batch_cases():
    for name in BATCH_GRAD_CASES:
        c = load_batch_grad_case(name)
        B, N = c["B"], c["points"].shape[2]
        assert c["grad32"].shape == c["grad64"].shape == (B, 3, N) and c["value"].shape == c["expected"].shape, name
        assert (c["value"] - c["expected"]).abs().max().item() < 2e-6, name
        assert (c["grad_output"] is not None) == (name == "c_rot"), name
    mixed = load_batch_grad_case("g_mixed")
    amax = [mixed["feat"][b].abs().max().item() for b in range(mixed["B"])]
    assert amax[1] > 12.0 and amax[0] < 12.0 and amax[2] < 12.0, amax
    # ragged against the 16-point tiles of the tensor-core program and the 8- to 32-point tiles of the exact kernel
    assert {load_batch_grad_case(n)["points"].shape[2] for n in BATCH_GRAD_CASES} == {1000, 2049, 515}


@pytest.mark.parametrize("name", BATCH_GRAD_CASES)
def test_restatement_matches_batch_grad_golden(name):
    c = load_batch_grad_case(name)
    for b in range(c["B"]):
        s = single(c, b)
        gout = s["grad_output"][0] if s["grad_output"] is not None else None
        _, g64 = query_grad_ref(s["feat"], s["points"], s["calib"], c["Ws"], c["bs"], c["last_op"], c["proj"], grad_output=gout,
                                dtype=torch.float64)
        assert (g64 - c["grad64"][b]).abs().max().item() <= 1e-9 * c["grad64"][b].abs().max().item(), (name, b)
        _, g32 = query_grad_ref(s["feat"], s["points"], s["calib"], c["Ws"], c["bs"], c["last_op"], c["proj"], grad_output=gout)
        ok, msg = within_bar(g32, c["grad32"][b])
        assert ok, (name, b, msg)


@pytest.mark.parametrize("name", ["g_nocalib", "c_small"])
@pytest.mark.parametrize("op", ["jvp", "grad"])
def test_batch_image_equals_single_launch_bit_for_bit(emu_tc, emu_fp32, tmp_path, name, op):
    """Image b of one batched launch == the single-map launch of image b (value and d points), in both programs and for both
    heads.  The tensor-core launch runs on 2 simulated SMs (tiles of both images on one CTA, the weight ring running across
    images) with the bulk copies completing in a random order."""
    c = _case(name)
    n = 37                                            # 3 tiles of 16 points per image, the last one ragged
    exe = emu_tc if op == "jvp" else emu_fp32
    env = {"EMU_TC_ORDER": "random:4"} if op == "jvp" else None
    got = _grad(exe, op, tmp_path, c, n, env=env, sms=2)
    for b in range(c["B"]):
        one = _grad(exe, op, tmp_path, single(c, b), n, batched=False, tag="one%d" % b, sms=2)
        assert torch.equal(got[0][b], one[0][0]) and torch.equal(got[1][b], one[1][0]), (name, op, b)
    assert bool(torch.isfinite(got[1]).all()) and got[1].abs().max().item() > 0


@pytest.mark.parametrize("sms", [1, 3])
def test_range_guard_per_image(emu_tc, emu_fp32, tmp_path, sms):
    """Three maps, only the middle one above the limit.  The tensor-core launch guarded in range finishes under a random
    completion order (the producer and the consumers skip the same image -- a disagreement would deadlock the weight ring),
    leaves that image's value and d points untouched and writes the other two as the unguarded launch does; the exact
    launch guarded out of range writes exactly that image, as the unguarded exact launch does."""
    c, amax = _mixed_case()
    n = 40
    got = _grad(emu_tc, "jvp", tmp_path, c, n, env={"EMU_TC_ORDER": "random:3"}, sms=sms, limit=12, guard="in")
    free = _grad(emu_tc, "jvp", tmp_path, c, n, tag="free", sms=sms)
    for part in (0, 1):
        assert bool((got[part][1] == -4242.0).all()), "the image above the limit must stay untouched"
        assert torch.equal(got[part][0], free[part][0]) and torch.equal(got[part][2], free[part][2])
    ex = _grad(emu_fp32, "grad", tmp_path, c, n, tag="ex", sms=sms, limit=12, guard="out", amax=_amax_option(c["feat"]))
    exfree = _grad(emu_fp32, "grad", tmp_path, c, n, tag="exfree", sms=sms)
    for part in (0, 1):
        assert bool((ex[part][0] == -4242.0).all()) and bool((ex[part][2] == -4242.0).all())
        assert torch.equal(ex[part][1], exfree[part][1])


@pytest.mark.parametrize("name", BATCH_GRAD_CASES)
def test_batched_programs_meet_the_batch_grad_golden_bars(emu_tc, emu_fp32, tmp_path, name):
    """The first 24 points of every image (the 8 border points, then a ragged 16-point tile): the exact launch against the
    reference's fp32 autograd (every component <= 1e-3 max|g|, 99 % <= 2e-5 max|g|); the MP_MODE_TC route -- the tensor-core
    launch guarded in range, then the exact launch guarded out of range, each image taken by one of them -- against its
    fp64 autograd (median <= 5e-5, p99 <= 5e-3, max <= 5e-2 of max|g|).  In g_mixed image 1 is above the geometry head's
    limit of 12 and is differentiated by the exact kernel.  Points outside the image get exactly 0."""
    c = load_batch_grad_case(name)
    n = 24
    limit = 12 if c["net"] == "G" else 8
    ex = _grad(emu_fp32, "grad", tmp_path, c, n, tag="ex")
    assert (ex[0] - c["value"][:, :, :n]).abs().max().item() <= 2e-5
    for b in range(c["B"]):
        ok, msg = within_bar(ex[1][b], c["grad32"][b, :, :n])
        assert ok, (b, msg)
    tc = _grad(emu_tc, "jvp", tmp_path, c, n, tag="tc", limit=limit, guard="in")
    out = _grad(emu_fp32, "grad", tmp_path, c, n, tag="out", limit=limit, guard="out", amax=_amax_option(c["feat"]))
    above = [c["feat"][b].abs().max().item() > limit for b in range(c["B"])]
    assert above == [name == "g_mixed" and b == 1 for b in range(c["B"])]
    val = torch.stack([out[0][b] if above[b] else tc[0][b] for b in range(c["B"])])
    dp = torch.stack([out[1][b] if above[b] else tc[1][b] for b in range(c["B"])])
    for b in range(c["B"]):
        skipped = (out if not above[b] else tc)
        assert bool((skipped[0][b] == -4242.0).all()) and bool((skipped[1][b] == -4242.0).all()), b
        if above[b]:
            assert torch.equal(val[b], ex[0][b]) and torch.equal(dp[b], ex[1][b]), b
    assert (val - c["value"][:, :, :n]).abs().max().item() <= 1e-4
    ok, msg = tc_bar(dp, c["grad64"][:, :, :n])
    print(name, msg)
    assert ok, msg
    outside = (c["value"][:, :, :n] == 0).all(1)
    for b in range(c["B"]):
        assert bool((dp[b][:, outside[b]] == 0).all()) and bool((ex[1][b][:, outside[b]] == 0).all()), b


# sha256 of out.f32 of `emu_tc jvp` on the first n points of the grad_* golden (value [Res,n], then d points [3,n]; 3
# simulated SMs), as the single-map program gave them before it covered a batch: a single map is a batch of one, and
# its bits did not move
SINGLE_MAP_BYTES = {
    ("g_nocalib", 50): "d0ac6481118f24c3ba0fbba6ad0cac568533ed31464be1355cef19c1dafa06c1",
    ("g_persp", 48): "adb5ff8947bb6a8938d151edbdd67960fdb28a939b5b157224d2bb3f3cf156bd",
    ("c_rot", 32): "1a0f22c7a5cb11484bb4cc9f556ed2aba9adfed578158388311ed4fef4c68760",
}


@pytest.mark.parametrize("name,n", sorted(SINGLE_MAP_BYTES))
def test_single_map_jvp_keeps_its_bytes(emu_tc, tmp_path, name, n):
    c = load_grad_case(name)
    gout = [] if c["grad_output"] is None else [c["grad_output"][:, :n].contiguous()]
    inp = dict(feat=c["feat"], rows=c["points"][:, :, :n], calib=c["calib"], proj=c["proj"], res=c["chans"][-1],
               last_op=c["last_op"], Ws=c["Ws"], bs=c["bs"])
    out, _ = run(emu_tc[0], tmp_path, "jvp", *gout, inp=inp, shape=None, options=dict(sms=3))
    assert hashlib.sha256(out).hexdigest() == SINGLE_MAP_BYTES[(name, n)]
