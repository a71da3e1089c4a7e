"""CPU model of the in-image grid launch (mp_launch_query_tc_grid in query_tc.cu, compiled unmodified by the grid-in-image
op of tests/emu/emu_tc.cpp): the ordered compaction lists the nodes of a grid range that project into the image and stores
+0 for the others, and the tensor-core program runs over the list.  The range must equal the dense MP_SRC_GRID launch bit
for bit, compared as int32 views so that the sign of zero counts."""
import numpy as np
import pytest

from emu_harness import build, needs_emu, run
from oracle import spec

pytestmark = needs_emu


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    return build(tmp_path_factory, "emu_tc")


def _bench_head_and_map():
    """bench.py's synthetic head, on its map pooled to 32 x 32 (the per-frame products of the CPU model stay cheap)"""
    import bench
    import torch
    _, Ws, bs, feats = bench.synthetic(n_feat=1)
    feat = torch.nn.functional.avg_pool2d(feats[0], 4)[0].numpy()
    return Ws, bs, feat


def _run(harness, tmp_path, calib, R, lin0, n, sms=3, feat_edit=None, peers=False):
    Ws, bs, feat = _bench_head_and_map()
    if feat_edit is not None:
        feat = feat_edit(feat.copy())
    inp = dict(feat=feat, rows=np.zeros((3, 1), np.float32), calib=calib, proj="orthogonal", res=1, last_op=spec.LAST_SIGMOID,
               Ws=Ws, bs=bs)
    out, r = run(harness, tmp_path, "grid-in-image", R, lin0, n, inp=inp, shape=(2, n), options=dict(sms=sms, peers=peers))
    out = out.numpy().view(np.int32)
    return out[0], out[1], int(r.stdout.split()[-1])


def _calib():
    import bench
    return bench.scene_calib().numpy()


# ranges of the bench camera that start and end inside a plane and cross the image's edge
@pytest.mark.parametrize("R,lin0,n,sms", [(33, 33 * 33 * 12 + 17, 1500, 3), (65, 65 * 65 * 5 + 7, 1500, 5)])
def test_bench_camera_equals_dense(harness, tmp_path, R, lin0, n, sms):
    dense, listed, in_img = _run(harness, tmp_path, _calib(), R, lin0, n, sms)
    assert 0 < in_img < n, in_img
    assert np.array_equal(dense, listed)
    assert int((listed == 0).sum()) >= n - in_img                 # +0 (bits 0) for every node outside the image


def test_peer_volumes_are_written_by_node_index(harness, tmp_path):
    dense, listed, in_img = _run(harness, tmp_path, _calib(), 33, 33 * 33 * 20 + 5, 1200, 4, peers=True)
    assert 0 < in_img < 1200
    assert np.array_equal(dense, listed)


def test_every_node_inside(harness, tmp_path):
    cal = _calib().copy()
    cal[0, :3, :] *= 0.25
    dense, listed, in_img = _run(harness, tmp_path, cal, 33, 33 * 33 * 7 + 3, 700)
    assert in_img == 700
    assert np.array_equal(dense, listed)


def test_every_node_outside_writes_zeros_only(harness, tmp_path):
    """an empty list: the program over it writes nothing, and every node holds the compaction's +0"""
    cal = _calib().copy()
    cal[0, 0, 3] += 10.0
    dense, listed, in_img = _run(harness, tmp_path, cal, 33, 33 * 33 * 7 + 3, 700, 2)
    assert in_img == 0
    assert np.array_equal(dense, listed) and not listed.any()


def test_map_with_a_nan_lists_every_node(harness, tmp_path):
    def poison(f):
        f[3, :, -1] = np.nan                      # the image's edge column: nodes just outside the image sample it too
        return f
    dense, listed, in_img = _run(harness, tmp_path, _calib(), 33, 33 * 33 * 12 + 17, 1500, 3, feat_edit=poison)
    assert 0 < in_img < 1500
    assert np.array_equal(dense, listed)
    assert np.isnan(dense.view(np.float32)).any()
