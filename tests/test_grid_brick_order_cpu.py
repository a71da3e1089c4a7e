"""CPU model of the brick order of the in-image list (mp_launch_query_tc_grid in query_tc.cu, compiled unmodified by
tests/emu/emu_query_grid_brick.cpp): the compaction scans a brick-major index space over the brick layers that the
range's z planes cross.  On ranges whose ends are not on a plane, it must list each in-image node of the range exactly
once, in 4x4x4-brick order, give every other node of the range +0, touch nothing else, and leave the volume of the
dense launch bit for bit."""
import struct
import subprocess

import numpy as np
import pytest

import emu_harness
from emu_harness import needs_emu, write_input
from oracle import spec
from tools.tile_texels import brick_order

emu_harness.HARNESSES.setdefault("emu_query_grid_brick", ("-O3", True))

pytestmark = needs_emu


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    return emu_harness.build(tmp_path_factory, "emu_query_grid_brick")


def _run(harness, tmp_path, R, lin0, n, sms=3, feat_edit=None):
    import bench
    import torch
    _, Ws, bs, feats = bench.synthetic(n_feat=1)
    feat = torch.nn.functional.avg_pool2d(feats[0], 4)[0].numpy()     # (a 32 x 32 map keeps the per-frame products cheap)
    if feat_edit is not None:
        feat = feat_edit(feat.copy())
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    write_input(fin, feat, np.zeros((3, 1), np.float32), bench.scene_calib().numpy(), "orthogonal", 1, spec.LAST_SIGMOID,
                Ws, bs)
    r = subprocess.run([harness, fin, fout, str(sms), str(R), str(lin0), str(n)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    raw = open(fout, "rb").read()
    count, size = struct.unpack("2q", raw[:16])
    assert 0 <= count <= n, count
    o = 16
    out = np.frombuffer(raw, np.int32, 2 * n, o).reshape(2, n)
    o += 8 * n
    lst = np.frombuffer(raw, np.int32, count, o).astype(np.int64)
    o += 4 * count
    visits = np.frombuffer(raw, np.int32, n, o)
    inside = np.frombuffer(raw, np.uint8, n, o + 4 * n).astype(bool)
    return out[0], out[1], lst, visits, inside, size


def _check(R, lin0, n, dense, listed, lst, visits, inside, size, every_node=False):
    layers = (lin0 + n - 1) // (R * R) // 4 - lin0 // (R * R) // 4 + 1
    assert size == layers * 64 * ((R + 3) // 4) ** 2              # the brick layers the range's z planes cross
    assert (visits == 1).all()                                    # each node of the range at exactly one index
    want = lin0 + np.arange(n) if every_node else lin0 + np.flatnonzero(inside)
    assert np.unique(lst).size == lst.size                        # no duplicates
    assert np.array_equal(np.sort(lst), want)                     # a permutation of the ascending in-image list
    assert np.array_equal(lst, brick_order(want, R))              # in brick order
    assert np.array_equal(dense, listed)                          # the dense launch, bit for bit (sign of zero included)
    if not every_node:
        assert not listed[~inside].any()                          # +0 outside the image


# the bench camera; ranges that start and end inside a plane and cross brick layers, a whole grid, a range inside one row
@pytest.mark.parametrize("R,lin0,n,sms", [
    (17, 0, 17 ** 3, 3),
    (17, 17 * 17 * 3 + 5, 17 * 17 * 6 + 11, 4),
    (33, 33 * 33 * 11 + 30, 1500, 3),
    (33, 33 * 33 * 16 + 33 * 10 + 4, 9, 2),
    (65, 65 * 65 * 7 + 100, 65 * 65 + 50, 5),
])
def test_brick_list_is_the_in_image_list(harness, tmp_path, R, lin0, n, sms):
    dense, listed, lst, visits, inside, size = _run(harness, tmp_path, R, lin0, n, sms)
    if n > 100:
        assert 0 < inside.sum() < n
    _check(R, lin0, n, dense, listed, lst, visits, inside, size)


def test_map_with_a_nan_lists_every_node_in_brick_order(harness, tmp_path):
    def poison(f):
        f[3, :, -1] = np.nan
        return f
    R, lin0, n = 33, 33 * 33 * 14 + 20, 1500
    dense, listed, lst, visits, inside, size = _run(harness, tmp_path, R, lin0, n, 3, feat_edit=poison)
    assert 0 < inside.sum() < n
    _check(R, lin0, n, dense, listed, lst, visits, inside, size, every_node=True)
    assert np.isnan(dense.view(np.float32)).any()
