"""The lossless engine (Seg3dLossless(faster=False)) inside the captured frame step: mp_octree_run_fused_async runs each
level's conflict loop as a conditional WHILE node decided on the device.  Against the host-driven mp_octree_run_fused it
must give the same volume, non-empty flag and per-level counts bit for bit, and as many passes per level as the generic
engine calls its query_func; FrameGraph / FrameGraphRing over lossless frames return exactly what the eager engine and
forward_vertices return, including the rendered images, and the 257^3 lossless property holds for a captured frame.  A
capture that succeeds is itself the check that the step never synchronises with the host."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import spec
from helpers import build_net

pytestmark = pytest.mark.gpu

B = np.array([[-1.0, -1.0, -1.0]], dtype=np.float32)
RES = [17, 33, 65, 129]


def _person(scale=1.0):
    Ws, bs = spec.make_weights(spec.G_CHANNELS, 3)
    base = spec.make_feat(256, 128, 128, 4, 0.5)
    W2, b2, f, _ = spec.heightfield_person(Ws, bs, base * scale, channel=0)
    return build_net("G", W2, b2), f.cuda()


def _ridge(feat):
    """A one-texel diagonal ridge of the height map, from the corner of the map into the left arm: a fin thinner than a
    voxel that the coarse levels miss and the conflict loop walks."""
    f = feat.clone()
    i = torch.arange(4, 60, device=f.device)
    f[0, 0, i, i] = 0.3
    return f


def _empty(feat):
    f = feat.clone()
    f[0, 0] = -5.0                                       # height map far below every node: nothing occupied
    return f


def _lossless(net, res=RES):
    from monoport_b200.engine import Seg3dLossless, make_query_func
    return Seg3dLossless(make_query_func(net), B, -B, res, balance_value=0.5, faster=False).to("cuda")


def _generic_passes(net, feat, cal, res=RES):
    """Passes per level the device loop must make: max(1, calls of query_func at that level) of the generic engine."""
    from monoport_b200.engine import Seg3dLossless
    sizes = []

    def plain(points, im_feat_list, calib_tensor):          # RTL/main.py:168-183 without the fused tag
        sizes.append(points.shape[1])
        return net.query(im_feat_list, points=points.permute(0, 2, 1), calibs=calib_tensor)[0]
    g = Seg3dLossless(plain, B, -B, res, balance_value=0.5, faster=False).to("cuda")
    g(im_feat_list=[[feat]], calib_tensor=cal)
    calls, k = [], 0
    for total in g.last_stats:                               # the calls come level after level, every one with points
        n = 0
        while total > 0:
            total -= sizes[k]
            k += 1
            n += 1
        calls.append(n)
    assert k == len(sizes)
    return [0] + [max(1, c) for c in calls[1:]]


def _run_async(eng, net, feat, cal):
    """mp_octree_run_fused_async on a fresh lossless handle, eager (the stream is not being captured)."""
    from monoport_b200 import _lib
    from monoport_b200.modeling.geometry import perspective
    lib = _lib.load()
    R = eng.resolutions[-1]
    n = len(eng.resolutions)
    h = eng._new_handle(torch.device("cuda"))
    out = torch.full((1, 1, R, R, R), -1.0, device="cuda")
    fh = net.feature_handle(feat)
    proj = _lib.PROJ_PERSPECTIVE if net.projection is perspective else _lib.PROJ_ORTHOGONAL
    st = _lib.stream_ptr()
    _lib.check(lib.mp_octree_run_fused_async(h, net.surface_classifier.handle(), fh.ptr, _lib.calib12(cal), proj,
                                             ctypes.c_float(net.normalizer.scale), net._mode(),
                                             ctypes.c_void_p(out.data_ptr()), st), "mp_octree_run_fused_async")
    nonempty = ctypes.c_int(0)
    stats = (ctypes.c_int64 * n)()
    loops = (ctypes.c_int32 * n)()
    _lib.check(lib.mp_octree_fetch(h, ctypes.byref(nonempty), stats, st), "mp_octree_fetch")
    _lib.check(lib.mp_octree_fetch_loops(h, loops, st), "mp_octree_fetch_loops")
    lib.mp_octree_destroy(h)
    return (out if nonempty.value else None), list(stats), list(loops)


@pytest.mark.parametrize("ridge", [False, True])
@pytest.mark.parametrize("precision", ["fp32", "tc", "auto"])
def test_async_lossless_equals_host_driven_loop(precision, ridge):
    net, feat = _person()
    if precision != "fp32" and not net.surface_classifier.tc_supported():
        pytest.skip("tensor-core program not supported")
    net.precision = precision
    if ridge:
        feat = _ridge(feat)
    cal = spec.scene_calib(20, 33).cuda()
    eng = _lossless(net)
    want = eng(im_feat_list=[[feat]], calib_tensor=cal)
    got, stats, loops = _run_async(eng, net, feat, cal)
    assert want is not None and got is not None
    assert torch.equal(got, want)
    assert stats == eng.last_stats, (stats, eng.last_stats)
    passes = _generic_passes(net, feat, cal)
    print("%s ridge=%s: passes per level %s, nodes per level %s" % (precision, ridge, loops, stats))
    assert loops == passes, (loops, passes)
    if ridge:
        assert loops[-1] >= 5, loops                     # the ridge is really walked


def test_frame_graph_ring_over_lossless_frames():
    """Two lanes, frames ridge, plain, empty, ridge: a replay that needs fewer passes after one that needs more, and an
    empty frame; every frame equals the eager engine + forward_vertices, stats and passes included."""
    from monoport_b200.pipeline import FrameGraph, FrameGraphRing
    from monoport_b200.recon import forward_vertices
    net, feat = _person()
    cal = spec.scene_calib(20, 33)
    frames = [_ridge(feat), feat, _empty(feat), _ridge(feat)]
    eng = _lossless(net)
    want = []
    for f in frames:
        sdf = eng(im_feat_list=[[f]], calib_tensor=cal.cuda())
        X, Y, Z, N = forward_vertices(sdf, "front")
        want.append((None if sdf is None else sdf.clone(), X, Y, Z, N, list(eng.last_stats),
                     _generic_passes(net, f, cal.cuda())))
    assert want[2][0] is None and want[0][0] is not None
    assert want[0][6][-1] > want[1][6][-1], "the ridge frame should need more passes than the plain one"
    ring = FrameGraphRing(lambda: FrameGraph(net, eng, cal, "front", with_encoder=False), n_lanes=2)
    n_out = 0
    for i, (w, out) in enumerate(zip(want, ring.run(iter(frames)))):
        n_out += 1
        lane = ring.lanes[i % 2]
        assert lane.last_stats == w[5], (i, lane.last_stats, w[5])
        assert lane.last_conflict_loops == w[6], (i, lane.last_conflict_loops, w[6])
        if w[0] is None:
            assert out[0] is None
            continue
        for a, b in zip(w[:5], out):
            assert torch.equal(a, b), i
    assert n_out == len(frames)
    ring.close()


def test_frame_graph_lossless_renders_colour_and_analytic_normals():
    """One lane with netC and render_normals="gradient" over lossless frames: the images equal eager colorization() and
    colorization(norm=surface_normals(precision="auto")) on the eager frame's vertices, bit for bit."""
    from monoport_b200.pipeline import FrameGraph
    from monoport_b200.recon import colorization, forward_vertices, surface_normals
    net, feat = _person()
    cal = spec.scene_calib(20, 33)
    Wc, bc = spec.make_weights(spec.C_CHANNELS, 21)
    netC = build_net("C", Wc, bc)
    c0 = spec.make_feat(512, 128, 128, 22, 0.5).cuda()
    eng = _lossless(net, [17, 33, 65])
    fg = FrameGraph(net, eng, cal, "front", with_encoder=False, netC=netC, render_normals="gradient")
    for f in (_ridge(feat), feat):
        sdf = eng(im_feat_list=[[f]], calib_tensor=cal.cuda())
        X, Y, Z, N = forward_vertices(sdf, "front")
        out = fg.launch(f, c0).result()
        rnorm, rtex = fg.rendered()
        assert fg.last_stats == eng.last_stats
        for a, b in zip((sdf, X, Y, Z, N), out):
            assert torch.equal(a, b)
        nrm = surface_normals(net, [[f]], X, Y, Z, cal.cuda(), resolution=65, precision="auto")
        assert torch.equal(rnorm, colorization(None, None, X, Y, Z, cal.cuda(), norm=nrm, resolution=65))
        assert torch.equal(rtex, colorization(netC, [[c0]], X, Y, Z, cal.cuda(), resolution=65))
    fg.close()


def test_lossless_property_of_a_captured_frame_at_full_size():
    """257^3: the captured lossless frame's mask equals the dense mask of the same net, its volume equals the eager
    engine's, and it evaluates a small fraction of the nodes."""
    from monoport_b200.pipeline import FrameGraph
    net, feat = _person()
    net.precision = "fp32"
    cal = spec.scene_calib(20, 33)
    res = [17, 33, 65, 129, 257]
    eng = _lossless(net, res)
    want = eng(im_feat_list=[[feat]], calib_tensor=cal.cuda())
    fg = FrameGraph(net, eng, cal, "front", with_encoder=False)
    sdf = fg.launch(feat).result()[0]
    assert sdf is not None and torch.equal(sdf, want)
    assert fg.last_stats == eng.last_stats
    dense = net.query_grid(feat, cal.cuda(), 257, torch.tensor([-1.0] * 3), torch.tensor([1.0] * 3))
    mism = int(((sdf[0, 0] > 0.5) != (dense > 0.5)).sum())
    print("257^3 captured lossless frame: %d nodes evaluated (%.2f%%), passes %s, mask mismatches %d"
          % (sum(fg.last_stats), 100.0 * sum(fg.last_stats) / 257 ** 3, fg.last_conflict_loops, mism))
    assert mism == 0
    assert sum(fg.last_stats) < 0.05 * 257 ** 3
    fg.close()
