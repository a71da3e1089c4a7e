"""A per-frame camera in the captured frame: FrameGraph reads its camera from a device buffer that launch(calib=...) rewrites
before every replay (the _dcal entry points).  Every frame of a ring driven through the demo's AUTO sequence (yaw 20 deg,
pitch 0, 3, 6, ...) and its FRONT / BACK / LEFT / RIGHT views (pitch 0, 180, 90, 270) equals the eager chain run with that
frame's camera bit for bit, for the three engines and for the whole frame (netC colour image, analytic normal image, mesh
with normals and colours); and each _dcal twin equals its by-value twin."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import spec
from helpers import build_net

pytestmark = pytest.mark.gpu

RES = [17, 33, 65]
AUTO = [spec.scene_calib(20, 3 * k) for k in range(6)]
VIEWS = [spec.scene_calib(20, p) for p in (0, 180, 90, 270)]


def _person(proj="orthogonal"):
    Ws, bs = spec.make_weights(spec.G_CHANNELS, 3)
    base = spec.make_feat(256, 128, 128, 4, 0.5)
    feats = []
    for k in range(2):
        W2, b2, f, _ = spec.heightfield_person(Ws, bs, base * (1.0 + 0.1 * k), channel=0)
        feats.append(f.cuda())
    return build_net("G", W2, b2, proj=proj), feats


def _out_of_image(cal):
    """a camera that moves the body out of the image: nothing is occupied"""
    c = cal.clone()
    c[0, 0, 3] += 10.0
    return c


def _engine(net, kind):
    from monoport_b200.engine import Seg3dLossless, Seg3dTopk, make_query_func
    b = np.array([[-1.0, -1.0, -1.0]], dtype=np.float32)
    if kind == "topk":
        return Seg3dTopk(make_query_func(net), b, -b, RES, [0, 9000, 30000]).to("cuda")
    return Seg3dLossless(make_query_func(net), b, -b, RES, balance_value=0.5, faster=kind == "faster").to("cuda")


def _same(a, b):
    if a is None or b is None:
        return a is None and b is None
    return a.shape == b.shape and bool(((a == b) | (torch.isnan(a) & torch.isnan(b))).all())


def _eager(eng, f, cal):
    from monoport_b200.recon import forward_vertices
    sdf = eng(im_feat_list=[[f]], calib_tensor=cal.cuda())
    sdf = None if sdf is None else sdf.clone()
    return (sdf,) + tuple(forward_vertices(sdf, "front")), list(eng.last_stats)


@pytest.mark.parametrize("kind", ["faster", "lossless", "topk"])
@pytest.mark.parametrize("lanes", [1, 2])
def test_ring_follows_the_demo_cameras(kind, lanes):
    """Ring frames over the AUTO sequence, the four views and an empty frame equal engine(calib_tensor=calib_k) +
    forward_vertices bit for bit, with the same last_stats."""
    from monoport_b200.pipeline import FrameGraph, FrameGraphRing
    net, feats = _person()
    eng = _engine(net, kind)
    cams = AUTO[:4] + [_out_of_image(AUTO[4])] + VIEWS
    frames = [feats[k % 2] for k in range(len(cams))]
    want = [_eager(eng, f, c) for f, c in zip(frames, cams)]
    assert want[4][0][0] is None and all(w[0][0] is not None for k, w in enumerate(want) if k != 4)
    ring = FrameGraphRing(lambda: FrameGraph(net, eng, VIEWS[2], "front", with_encoder=False), n_lanes=lanes)
    n = 0
    for i, ((w, stats), out) in enumerate(zip(want, ring.run(iter(frames), calibs=cams))):
        n += 1
        for k, (a, b) in enumerate(zip(w, out)):
            assert _same(a, b), (kind, i, k)
        assert ring.lanes[i % lanes].last_stats == stats, (kind, i)
    assert n == len(cams)
    ring.close()


def test_graph_built_with_a_and_launched_with_b_is_the_graph_built_with_b():
    """The lossless engine (conflict loops in WHILE nodes): a graph captured with camera A and launched with camera B gives
    what a graph captured with B gives -- volume, vertices, last_stats and last_conflict_loops; launch() without a calib
    after that gives A again; a CPU calib changed right after launch() and a CUDA calib produced on the caller's stream are
    the frame's camera."""
    from monoport_b200.pipeline import FrameGraph
    net, feats = _person()
    eng = _engine(net, "lossless")
    a, b = AUTO[0], VIEWS[2]
    ga = FrameGraph(net, eng, a, "front", with_encoder=False)
    gb = FrameGraph(net, eng, b, "front", with_encoder=False)

    def run(g, **kw):
        out = g.launch(feats[0], **kw).result()
        return tuple(None if t is None else t.clone() for t in out), g.last_stats, g.last_conflict_loops

    want_b, want_a = run(gb), run(ga)
    assert sum(want_b[2]) > 0
    got = run(ga, calib=b)
    assert all(_same(x, y) for x, y in zip(got[0], want_b[0])) and got[1:] == want_b[1:]
    got = run(ga)                                                  # calib=None: the constructor's camera
    assert all(_same(x, y) for x, y in zip(got[0], want_a[0])) and got[1:] == want_a[1:]
    # a CPU tensor the caller changes as soon as launch() returns
    cpu = b.clone()
    torch.cuda._sleep(20_000_000)                                  # keep the device busy: the replay is still ahead
    ga.launch(feats[0], calib=cpu)
    cpu.copy_(a)
    out = ga.result()
    assert all(_same(x, y) for x, y in zip(out, want_b[0]))
    # a CUDA calib produced on the caller's stream just before launch(), float64 and [4,4]
    torch.cuda._sleep(20_000_000)
    dev = b[0].cuda().double() * 1.0
    out = ga.launch(feats[0], calib=dev).result()
    assert all(_same(x, y) for x, y in zip(out, want_b[0]))
    ga.close()
    gb.close()


def test_whole_frame_follows_the_camera():
    """netC, the analytic normal image and the mesh with normals and colours: every output of every frame equals its eager
    twin with that frame's camera -- including a frame above the geometry head's feature limit (the exact route) and an empty
    frame."""
    from monoport_b200.pipeline import FrameGraph, FrameGraphRing
    from monoport_b200.recon import colorization, forward_vertices, mesh_colours, mesh_normals, reconstruction, surface_normals
    net, feats = _person()
    netC = build_net("C", *spec.make_weights(spec.C_CHANNELS, 21))
    eng = _engine(net, "faster")
    c0 = spec.make_feat(512, 128, 128, 22, 0.5).cuda()
    big = feats[1].clone()
    big[0, 7, 0, 0] = 40.0                               # above the head's limit: the exact kernels take this frame
    frames = [(feats[0], c0), (big, c0), (feats[1], c0), (feats[0], c0), (feats[1], c0)]
    cams = [AUTO[1], VIEWS[1], _out_of_image(AUTO[2]), VIEWS[3], AUTO[5]]
    R, b0, b1 = RES[-1], (-1.0, -1.0, -1.0), (1.0, 1.0, 1.0)
    want = []
    for (f, c), cal in zip(frames, cams):
        cal = cal.cuda()
        sdf = eng(im_feat_list=[[f]], calib_tensor=cal)
        if sdf is None:
            want.append(None)
            continue
        sdf = sdf.clone()
        X, Y, Z, N = forward_vertices(sdf, "front")
        Ng = surface_normals(net, [[f]], X, Y, Z, cal, R, b0, b1, precision="auto")
        rnorm = colorization(netC, None, X, Y, Z, cal, norm=Ng, resolution=R)
        rtex = colorization(netC, [[c]], X, Y, Z, cal, resolution=R)
        verts, faces, _, _ = reconstruction(net, "cuda", cal, R, b0, b1, use_octree=True, feats=[[f]], engine=eng)
        want.append((sdf, X, Y, Z, N, rnorm, rtex, verts, faces, mesh_normals(net, [[f]], verts, cal, "auto"),
                     mesh_colours(netC, [[c]], verts, cal)))
    assert want[2] is None and all(w is not None for k, w in enumerate(want) if k != 2)
    ring = FrameGraphRing(lambda: FrameGraph(net, eng, AUTO[0], "front", with_encoder=False, netC=netC, render_normals="gradient",
                                             mesh=True, mesh_normals=True, mesh_colours=True), n_lanes=2)
    for i, (w, out) in enumerate(zip(want, ring.run(iter(frames), calibs=cams))):
        if w is None:
            assert all(t is None for t in out)
            continue
        for k, (a, b) in enumerate(zip(w, out)):
            assert _same(a, b), (i, k)
    ring.close()


def test_perspective_net_follows_the_camera():
    from monoport_b200.pipeline import FrameGraph, FrameGraphRing
    net, feats = _person("perspective")
    eng = _engine(net, "lossless")
    cams = [AUTO[0], AUTO[3], VIEWS[1]]
    want = [_eager(eng, feats[0], c) for c in cams]
    ring = FrameGraphRing(lambda: FrameGraph(net, eng, AUTO[2], "front", with_encoder=False), n_lanes=2)
    for i, ((w, stats), out) in enumerate(zip(want, ring.run([feats[0]] * 3, calibs=cams))):
        assert all(_same(a, b) for a, b in zip(w, out)), i
        assert ring.lanes[i % 2].last_stats == stats
    ring.close()


def test_launch_refuses_a_bad_calib():
    from monoport_b200.pipeline import FrameGraph
    net, feats = _person()
    g = FrameGraph(net, _engine(net, "faster"), AUTO[0], "front", with_encoder=False)
    for bad in (torch.eye(4)[None].repeat(2, 1, 1), torch.eye(3), torch.zeros(4, 3), torch.eye(4, dtype=torch.int64),
                torch.eye(4)[None, None]):
        with pytest.raises(ValueError):
            g.launch(feats[0], calib=bad)
    if torch.cuda.device_count() > 1:
        with pytest.raises(ValueError):
            g.launch(feats[0], calib=torch.eye(4, device="cuda:1"))
    with pytest.raises(ValueError):
        g.launch(feats[0], calib=torch.eye(4, device="meta"))
    g.close()


# ---- the C ABI directly ------------------------------------------------------------------------------------------------------
def _p(t):
    return ctypes.c_void_p(t.data_ptr())


@pytest.mark.parametrize("kind", ["faster", "lossless"])
def test_octree_twin_off_capture(kind):
    """mp_octree_run_fused_async_dcal on a stream that is not being captured equals mp_octree_run_fused_async."""
    from monoport_b200 import _lib
    from monoport_b200.modeling.MonoPortNet import FeatureHandle
    lib = _lib.load()
    net, feats = _person()
    eng = _engine(net, kind)
    fh = FeatureHandle(256, 128, 128, torch.device("cuda"))
    fh.upload(feats[0])
    R = RES[-1]
    cal = VIEWS[2]
    cal_dev = cal[0, :3, :4].contiguous().cuda()
    head, st, z = net.surface_classifier.handle(), _lib.stream_ptr(), ctypes.c_float(net.normalizer.scale)
    outs = []
    for dcal in (False, True):
        oct_ = eng._new_handle(torch.device("cuda"))
        vol = torch.full((R, R, R), -7.0, device="cuda")
        if dcal:
            rc = lib.mp_octree_run_fused_async_dcal(oct_, head, fh.ptr, _p(cal_dev), _lib.PROJ_ORTHOGONAL, z, net._mode(), _p(vol), st)
        else:
            rc = lib.mp_octree_run_fused_async(oct_, head, fh.ptr, _lib.calib12(cal), _lib.PROJ_ORTHOGONAL, z, net._mode(), _p(vol), st)
        _lib.check(rc, "run")
        ne, stats = ctypes.c_int(0), (ctypes.c_int64 * 3)()
        _lib.check(lib.mp_octree_fetch(oct_, ctypes.byref(ne), stats, st), "fetch")
        outs.append((vol.clone(), ne.value, list(stats)))
        lib.mp_octree_destroy(oct_)
    assert outs[0][1] == 1 and outs[0][1:] == outs[1][1:]
    assert torch.equal(outs[0][0], outs[1][0])
    # refusals: no camera, and what the by-value call refuses (a head with 3 outputs)
    oct_ = eng._new_handle(torch.device("cuda"))
    vol = torch.empty((R, R, R), device="cuda")
    assert lib.mp_octree_run_fused_async_dcal(oct_, head, fh.ptr, None, 0, z, net._mode(), _p(vol), st) != 0
    netC = build_net("C", *spec.make_weights(spec.C_CHANNELS, 21))
    for fn, c in ((lib.mp_octree_run_fused_async, _lib.calib12(cal)), (lib.mp_octree_run_fused_async_dcal, _p(cal_dev))):
        assert fn(oct_, netC.surface_classifier.handle(), fh.ptr, c, 0, z, net._mode(), _p(vol), st) != 0
    lib.mp_octree_destroy(oct_)


@pytest.mark.parametrize("mode", ["fp32", "tc"])
def test_point_twins_equal_their_by_value_calls(mode):
    """mp_query_points_count_dcal, mp_mesh_normals_async_dcal, mp_surface_normals_async_dcal and
    mp_colorize_surface_async_dcal against their by-value twins, bit for bit; and their refusals."""
    from monoport_b200 import _lib
    from monoport_b200.modeling.MonoPortNet import FeatureHandle
    lib = _lib.load()
    net, feats = _person()
    netC = build_net("C", *spec.make_weights(spec.C_CHANNELS, 21))
    m = _lib.MODE_FP32 if mode == "fp32" else _lib.MODE_AUTO
    fh, fc = FeatureHandle(256, 128, 128, torch.device("cuda")), FeatureHandle(512, 128, 128, torch.device("cuda"))
    fh.upload(feats[0])
    fc.upload(spec.make_feat(512, 128, 128, 22, 0.5).cuda())
    cal = AUTO[4]
    c12, cdev = _lib.calib12(cal), cal[0, :3, :4].contiguous().cuda()
    st, zs = _lib.stream_ptr(), ctypes.c_float(net.normalizer.scale)
    g, hc = net.surface_classifier.handle(), netC.surface_classifier.handle()
    n = 3000
    pts = (torch.rand(n, 3, device="cuda") * 2 - 1).contiguous()
    cnt32 = torch.tensor([n - 17], dtype=torch.int32, device="cuda")
    cnt64 = torch.tensor([n - 17, 0], dtype=torch.int64, device="cuda")
    R = 65
    cols = torch.randperm(R * R, device="cuda")[:n // 2]
    X, Y = (cols // R).contiguous(), (cols % R).contiguous()
    Z = (torch.rand(n // 2, device="cuda") * (R - 1)).contiguous()
    vcnt = torch.tensor([n // 2 - 3], dtype=torch.int64, device="cuda")
    b0, b1 = _lib.f3([-1, -1, -1]), _lib.f3([1, 1, 1])

    def both(call):
        outs = [call(c12, False), call(_p(cdev), True)]
        torch.cuda.synchronize()
        for a, b in zip(outs[0], outs[1]):
            assert _same(a, b)

    def q(c, d):
        out = torch.full((3, n), -3.0, device="cuda")
        fn = lib.mp_query_points_count_dcal if d else lib.mp_query_points_count
        _lib.check(fn(hc, fc.ptr, _p(pts), n, 1, 3, c, 0, zs, _p(out), n, _p(cnt32), m, st), "q")
        return (out,)

    def mn(c, d):
        norm = torch.full((n, 3), -3.0, device="cuda")
        scratch = torch.empty(3 * n, device="cuda")
        fn = lib.mp_mesh_normals_async_dcal if d else lib.mp_mesh_normals_async
        _lib.check(fn(g, fh.ptr, _p(pts), _p(cnt64), _p(cnt32), n, c, 0, zs, m, _p(scratch), _p(norm), st), "mn")
        return (norm,)

    def sn(c, d):
        cap = n // 2
        norm = torch.full((cap, 3), -3.0, device="cuda")
        scratch = torch.empty(6 * cap + 1, device="cuda")
        fn = lib.mp_surface_normals_async_dcal if d else lib.mp_surface_normals_async
        _lib.check(fn(g, fh.ptr, _p(X), _p(Y), _p(Z), _p(vcnt), cap, R, b0, b1, c, 0, zs, m, _p(scratch), _p(norm), st), "sn")
        return (norm,)

    def cs(c, d):
        canvas = torch.ones((R, R, 3), device="cuda")
        fn = lib.mp_colorize_surface_async_dcal if d else lib.mp_colorize_surface_async
        _lib.check(fn(hc, fc.ptr, _p(X), _p(Y), _p(Z), _p(vcnt), n // 2, R, b0, b1, c, 0, zs, m, _p(canvas), st), "cs")
        return (canvas,)

    for call in (q, mn, sn, cs):
        both(call)
    # refusals: no camera; and what the twins refuse (a head with the wrong output count, a batched feature handle)
    scratch, out = torch.empty(6 * n + 1, device="cuda"), torch.empty((n, 3), device="cuda")
    assert lib.mp_query_points_count_dcal(hc, fc.ptr, _p(pts), n, 1, 3, None, 0, zs, _p(out), n, _p(cnt32), m, st) != 0
    assert lib.mp_mesh_normals_async_dcal(hc, fc.ptr, _p(pts), _p(cnt64), _p(cnt32), n, _p(cdev), 0, zs, m, _p(scratch),
                                          _p(out), st) != 0
    assert lib.mp_mesh_normals_async(hc, fc.ptr, _p(pts), _p(cnt64), _p(cnt32), n, c12, 0, zs, m, _p(scratch), _p(out), st) != 0
    assert lib.mp_surface_normals_async_dcal(hc, fc.ptr, _p(X), _p(Y), _p(Z), _p(vcnt), n // 2, R, b0, b1, _p(cdev), 0, zs, m,
                                             _p(scratch), _p(out), st) != 0
    assert lib.mp_colorize_surface_async_dcal(g, fh.ptr, _p(X), _p(Y), _p(Z), _p(vcnt), n // 2, R, b0, b1, _p(cdev), 0, zs, m,
                                              _p(out), st) != 0
    fb = FeatureHandle(512, 128, 128, torch.device("cuda"), B=2)
    assert lib.mp_query_points_count_dcal(hc, fb.ptr, _p(pts), n, 1, 3, _p(cdev), 0, zs, _p(out), n, _p(cnt32), m, st) != 0
    assert lib.mp_query_points_count(hc, fb.ptr, _p(pts), n, 1, 3, c12, 0, zs, _p(out), n, _p(cnt32), m, st) != 0
    torch.cuda.synchronize()
