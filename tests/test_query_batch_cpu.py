"""CPU checks of the batched query (mp_query_points_batch: B images in one launch): the oracle against the batched goldens of
the reference, and both query kernels -- compiled unmodified on the CPU model of tests/emu -- against those goldens and
against B = 1 runs of each image, bit for bit, including the per-image range guard of the tensor-core program."""
import pytest
import torch

from oracle import spec
from batch_cases import batch_cases, load_batch_case
from emu_harness import build, run


@pytest.mark.parametrize("name", batch_cases())
def test_oracle_per_image_matches_batched_reference_golden(name):
    c = load_batch_case(name)
    assert c["expected"].shape[0] == c["B"] and c["B"] >= 2
    for b in range(c["B"]):
        cal = c["calib"][b:b + 1] if c["calib"] is not None else None
        want = spec.query_ref(c["feat"][b], c["points"][b], cal, c["Ws"], c["bs"], c["last_op"], c["proj"])
        assert (want - c["expected"][b]).abs().max().item() < 2e-6, (name, b)


def test_batched_goldens_cover_the_issue_cases():
    assert set(batch_cases()) >= {"g_rot", "g_persp", "g_nocalib", "g_mixed", "c_rot"}
    mixed = load_batch_case("g_mixed")
    amax = [mixed["feat"][b].abs().max().item() for b in range(mixed["B"])]
    assert amax[1] > 12.0 and amax[0] < 12.0 and amax[2] < 12.0, amax


# ---- the kernels on the CPU model ------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu_tc(tmp_path_factory):
    return build(tmp_path_factory, "emu_tc")


@pytest.fixture(scope="module")
def emu_fp32(tmp_path_factory):
    return build(tmp_path_factory, "emu_fp32")


def _run(exe, tmp_path, case, n, batched, env=None, feat=None, tag="x", **options):
    """-> [B,Res,n] (a batched launch of every image of the case) or [Res,n] (a single-image launch)"""
    feat = case["feat"] if feat is None else feat
    res = case["expected"].shape[1]
    inp = dict(feat=feat, rows=case["points"][:, :, :n], calib=case["calib"], proj=case["proj"], res=res,
               last_op=case["last_op"], Ws=case["Ws"], bs=case["bs"], batched=batched)
    B = feat.shape[0]
    return run(exe, tmp_path, "query", inp=inp, shape=(B, res, n) if batched else (res, n),
               options=dict(batch=B if batched else None, **options), env=env, tag=tag)[0]


def _single(case, b):
    """image b of a batched case as a B = 1 case"""
    c = dict(case)
    c["feat"] = case["feat"][b:b + 1]
    c["points"] = case["points"][b:b + 1]
    c["calib"] = case["calib"][b:b + 1] if case["calib"] is not None else None
    return c


@pytest.mark.parametrize("name,n,sms", [
    ("g_nocalib", 150, 2),       # 32 x 32 maps, calibs=None, ragged last tile of every image
    ("g_persp", 70, 3),          # perspective: one full and one 6-point tile per image
    ("c_rot", 66, 1),            # colour head: one CTA walks all tiles of both images (ring across images)
])
def test_tc_batch_matches_batched_reference_golden(emu_tc, tmp_path, name, n, sms):
    c = load_batch_case(name)
    got = _run(emu_tc, tmp_path, c, n, True, sms=sms)
    want = c["expected"][:, :, :n]
    assert (got - want).abs().max().item() <= 1e-4
    assert torch.equal(got[want == 0], want[want == 0]), "out-of-image points must be exactly 0"


@pytest.mark.parametrize("name,n", [("g_nocalib", 150), ("g_persp", 70), ("c_rot", 40), ("g_rot", 33)])
def test_fp32_batch_matches_batched_reference_golden(emu_fp32, tmp_path, name, n):
    c = load_batch_case(name)
    got = _run(emu_fp32, tmp_path, c, n, True)
    want = c["expected"][:, :, :n]
    assert (got - want).abs().max().item() <= 2e-5
    assert torch.equal(got[want == 0], want[want == 0])


def test_fp32_batch_image_equals_single_run(emu_fp32, tmp_path):
    c = load_batch_case("g_nocalib")
    n = 77
    got = _run(emu_fp32, tmp_path, c, n, True)
    for b in range(c["B"]):
        one = _run(emu_fp32, tmp_path, _single(c, b), n, False, tag="one%d" % b)
        assert torch.equal(got[b], one), b


@pytest.mark.parametrize("sms", [1, 2, 3])
def test_tc_batch_image_equals_single_run_bit_for_bit(emu_tc, tmp_path, sms):
    """Image b of one batched launch == a B = 1 launch of image b, for 1, 2 and 3 simulated SMs (tiles of different images
    on one CTA, the weight ring running across images)."""
    c = load_batch_case("g_nocalib")
    n = 130
    got = _run(emu_tc, tmp_path, c, n, True, sms=sms)
    for b in range(c["B"]):
        one = _run(emu_tc, tmp_path, _single(c, b), n, False, tag="one%d" % b, sms=sms)
        assert torch.equal(got[b], one), (sms, b)


@pytest.mark.parametrize("order", ["random:1", "random:2"])
def test_tc_batch_bit_identity_under_other_completion_orders(emu_tc, tmp_path, order):
    c = load_batch_case("g_nocalib")
    n = 100
    want = _run(emu_tc, tmp_path, c, n, True, sms=2)
    got = _run(emu_tc, tmp_path, c, n, True, env={"EMU_TC_ORDER": order}, tag="ord", sms=2)
    assert torch.equal(got, want)
    for b in range(c["B"]):
        one = _run(emu_tc, tmp_path, _single(c, b), n, False, env={"EMU_TC_ORDER": order}, tag="one%d" % b, sms=2)
        assert torch.equal(got[b], one), b


@pytest.mark.parametrize("sms", [1, 3])
def test_tc_batch_range_guard_skips_exactly_the_out_of_range_image(emu_tc, tmp_path, sms):
    """Three 32 x 32 maps, the middle one scaled x4 so that exactly it is above the limit: the guarded tensor-core launch
    finishes (the producer and the consumers skip the same tiles -- a disagreement would deadlock the weight ring), leaves
    that image's sentinel outputs untouched and produces the other two images exactly."""
    c = load_batch_case("g_nocalib")
    feat = torch.cat([c["feat"][0:1], c["feat"][1:2] * 4.0, c["feat"][0:1] * 0.5], 0)
    pts = torch.cat([c["points"], c["points"][0:1].flip(2)], 0)
    case = dict(c, feat=feat, points=pts, B=3)
    amax = [feat[b].abs().max().item() for b in range(3)]
    limit = 12.0
    assert amax[1] > limit and amax[0] < limit and amax[2] < limit, amax
    n = 140
    got = _run(emu_tc, tmp_path, case, n, True, sms=sms, limit=limit, guard="in")
    assert bool((got[1] == -4242.0).all()), "the out-of-range image's outputs must stay untouched"
    free = _run(emu_tc, tmp_path, case, n, True, tag="free", sms=sms)      # no guard
    assert torch.equal(got[0], free[0]) and torch.equal(got[2], free[2])
    for b in (0, 2):
        one = _run(emu_tc, tmp_path, _single(case, b), n, False, tag="one%d" % b, sms=sms)
        assert torch.equal(got[b], one), b
