"""The mesh inside the captured frame step: the enqueue-only marching cubes (marching_cubes_async / mp_mcubes_run_async)
against marching_cubes() and reconstruction(), a FrameGraph(mesh=True, mesh_normals=True, mesh_colours=True) frame sequence
against the eager chain engine -> reconstruction -> mesh_normals -> mesh_colours, the exact mesh normals against
reconstruction(normals=True), capacity overflow, and the refusals of the new entry points.  A capture that succeeds is itself
the check that the step never synchronises with the host."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import spec
from helpers import build_net

pytestmark = pytest.mark.gpu

B_MIN, B_MAX = (-1.0, -1.0, -1.0), (1.0, 1.0, 1.0)
B = np.array([[-1.0, -1.0, -1.0]], dtype=np.float32)


def _person_frames():
    Ws, bs = spec.make_weights(spec.G_CHANNELS, 3)
    base = spec.make_feat(256, 128, 128, 4, 0.5)
    feats = []
    for k in range(3):
        W2, b2, f, _ = spec.heightfield_person(Ws, bs, base * (1.0 + 0.1 * k), channel=0)
        feats.append(f.cuda())
    return build_net("G", W2, b2), feats


def _engine(net, faster, res=(17, 33, 65)):
    from monoport_b200.engine import Seg3dLossless, make_query_func
    return Seg3dLossless(make_query_func(net), B, -B, list(res), balance_value=0.5, faster=faster).to("cuda")


def _colour_net():
    Wc, bc = spec.make_weights(spec.C_CHANNELS, 21)
    return build_net("C", Wc, bc)


def _buffers(v_cap, f_cap, guard=0):
    """output buffers of marching_cubes_async with `guard` sentinel rows behind the capacities"""
    vb = torch.full((v_cap + guard, 3), -12345.0, device="cuda")
    fb = torch.full((f_cap + guard, 3), -7, dtype=torch.int32, device="cuda")
    counts = torch.full((2,), -1, dtype=torch.int64, device="cuda")
    c32 = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    return vb, fb, counts, c32


def test_async_equals_marching_cubes_and_reconstruction():
    """Index space: marching_cubes() bit for bit.  World space: reconstruction(use_octree=True, engine=...)'s vertices and
    faces bit for bit.  One workspace, two volumes in turn."""
    from monoport_b200.recon import McubesWorkspace, marching_cubes, marching_cubes_async, reconstruction
    net, feats = _person_frames()
    cal = spec.scene_calib(20, 33).cuda()
    eng = _engine(net, True)
    ws = McubesWorkspace((65, 65, 65), "cuda")
    for f in feats[:2]:
        sdf = eng(im_feat_list=[[f]], calib_tensor=cal)
        vol = sdf[0, 0].clone()
        V, F = marching_cubes(vol)
        cap = 8 * 65 * 65
        vb, fb, counts, c32 = _buffers(cap, 2 * cap)
        marching_cubes_async(vol, vb, fb, counts, c32, workspace=ws)
        torch.cuda.synchronize()
        nv, nf = counts.tolist()
        assert (nv, nf) == (V.shape[0], F.shape[0]) and c32.item() == nv and nv > 0
        assert torch.equal(vb[:nv], V) and torch.equal(fb[:nf], F)
        Vw, Fw, _, _ = reconstruction(net, "cuda", cal, 65, B_MIN, B_MAX, use_octree=True, feats=[[f]], engine=eng)
        marching_cubes_async(vol, vb, fb, counts, c32, b_min=B_MIN, b_max=B_MAX, workspace=ws)
        torch.cuda.synchronize()
        assert counts.tolist() == [Vw.shape[0], Fw.shape[0]]
        assert torch.equal(vb[:nv], Vw) and torch.equal(fb[:nf], Fw)
    ws.close()


def test_capacity_overflow_leaves_the_guard_rows_and_raises_from_mesh():
    from monoport_b200.pipeline import FrameGraph
    from monoport_b200.recon import McubesWorkspace, marching_cubes, marching_cubes_async
    net, feats = _person_frames()
    cal = spec.scene_calib(20, 33)
    eng = _engine(net, True)
    vol = eng(im_feat_list=[[feats[0]]], calib_tensor=cal.cuda())[0, 0].clone()
    V, F = marching_cubes(vol)
    nV, nF = V.shape[0], F.shape[0]
    ws = McubesWorkspace(vol.shape, "cuda")
    for vc, fc in [(nV - 1, nF), (nV, nF - 1), (0, 0)]:
        vb, fb, counts, c32 = _buffers(vc, fc, guard=64)
        marching_cubes_async(vol, vb[:vc], fb[:fc], counts, c32, workspace=ws)
        torch.cuda.synchronize()
        assert counts.tolist() == [nV, nF] and c32.item() == min(nV, vc)
        assert torch.equal(vb[:vc], V[:vc]) and torch.equal(fb[:fc], F[:fc])
        assert bool((vb[vc:] == -12345.0).all()) and bool((fb[fc:] == -7).all()), (vc, fc)
    ws.close()
    fg = FrameGraph(net, eng, cal, "front", with_encoder=False, mesh=True, mesh_capacity=(nV - 1, nF))
    out = fg.launch(feats[0]).result()
    assert out[0] is not None
    with pytest.raises(RuntimeError, match="reconstruction"):
        fg.mesh()
    fg.close()


@pytest.mark.parametrize("n_lanes", [1, 2])
@pytest.mark.parametrize("faster", [True, False])
def test_captured_mesh_frames_equal_the_eager_chain(faster, n_lanes):
    """Frames: the person, the person with a ridge (another mesh), an empty frame, a third person whose colour map is above
    netC's feature limit (forced low: the exact kernel runs, decided on the device), the first again.  Every frame's mesh, normals and colours
    equal engine -> reconstruction -> mesh_normals("auto") -> mesh_colours bit for bit."""
    from monoport_b200.pipeline import FrameGraph, FrameGraphRing
    from monoport_b200.recon import mesh_colours, mesh_normals, reconstruction
    net, feats = _person_frames()
    netC = _colour_net()
    cal = spec.scene_calib(20, 33)
    eng = _engine(net, faster)
    c0 = spec.make_feat(512, 128, 128, 22, 0.5).cuda()
    c1 = spec.make_feat(512, 128, 128, 23, 0.5).cuda()
    limit = 1.5 * max(c0.abs().max().item(), c1.abs().max().item())
    netC.surface_classifier.tc_feature_limit = limit
    big = c0 * 4.0
    assert big.abs().max().item() > limit
    empty = feats[0].clone()
    empty[0, 0] = -5.0
    ridge = feats[1].clone()                             # a one-texel ridge of the height map: a different mesh
    d = torch.arange(4, 60, device=ridge.device)
    ridge[0, 0, d, d] = 0.3
    frames = [(feats[0], c0), (ridge, c1), (empty, c0), (feats[2], big), (feats[0], c1)]
    want = []
    for f, c in frames:
        r = reconstruction(net, "cuda", cal.cuda(), 65, B_MIN, B_MAX, use_octree=True, feats=[[f]], engine=eng)
        if isinstance(r, int):
            want.append(None)
            continue
        verts, faces, _, _ = r
        want.append((verts, faces, mesh_normals(net, [[f]], verts, cal.cuda(), precision="auto"),
                     mesh_colours(netC, [[c]], verts, cal.cuda())))
    assert want[2] is None and all(w is not None for k, w in enumerate(want) if k != 2)
    assert want[1][0].shape != want[0][0].shape
    ring = FrameGraphRing(lambda: FrameGraph(net, eng, cal, "front", with_encoder=False, netC=netC, mesh=True,
                                             mesh_normals=True, mesh_colours=True), n_lanes=n_lanes)
    n_out = 0
    for i, (w, out) in enumerate(zip(want, ring.run(iter(frames)))):
        n_out += 1
        assert len(out) == 11
        if w is None:
            assert all(t is None for t in out)
            continue
        for name, a, b in zip(("verts", "faces", "normals", "colours"), w, out[7:]):
            assert a.shape == b.shape and torch.equal(a, b), (i, name)
        print("frame %d: %d vertices, %d faces" % (i, w[0].shape[0], w[1].shape[0]))
    assert n_out == len(frames)
    ring.close()


def test_exact_mesh_normals_match_reconstruction_normals():
    """precision="fp32": the same exact gradient as reconstruction(normals=True); only the normalisation differs (torch's
    norm and division against the kernel's)."""
    from monoport_b200.recon import mesh_normals, reconstruction
    net, feats = _person_frames()
    cal = spec.scene_calib(20, 33).cuda()
    eng = _engine(net, True)
    verts, _, nrm, _ = reconstruction(net, "cuda", cal, 65, B_MIN, B_MAX, use_octree=True, feats=[[feats[0]]], engine=eng,
                                      normals=True)
    got = mesh_normals(net, [[feats[0]]], verts, cal, precision="fp32")
    err = (got - nrm).abs().max().item()
    print("mesh_normals(fp32) vs reconstruction(normals=True): max diff %.3e over %d vertices" % (err, verts.shape[0]))
    assert err <= 1e-6


def test_mesh_on_changes_no_other_output():
    """result() and rendered() of a graph with the mesh on equal those of one without; the ring's tuple grows by four."""
    from monoport_b200.pipeline import FrameGraph, FrameGraphRing
    net, feats = _person_frames()
    netC = _colour_net()
    cal = spec.scene_calib(20, 33)
    eng = _engine(net, True)
    c0 = spec.make_feat(512, 128, 128, 22, 0.5).cuda()
    frames = [(f, c0) for f in feats]
    plain = FrameGraphRing(lambda: FrameGraph(net, eng, cal, "front", with_encoder=False, netC=netC, render_normals="gradient"),
                           n_lanes=2)
    want = [tuple(None if t is None else t.clone() for t in out) for out in plain.run(iter(frames))]
    plain.close()
    ring = FrameGraphRing(lambda: FrameGraph(net, eng, cal, "front", with_encoder=False, netC=netC, render_normals="gradient",
                                             mesh=True, mesh_colours=True), n_lanes=2)
    for w, out in zip(want, ring.run(iter(frames))):
        assert len(w) == 7 and len(out) == 11
        for a, b in zip(w, out[:7]):
            assert torch.equal(a, b)
        assert out[9] is None and out[10] is not None           # normals off, colours on
    ring.close()


def test_new_entry_points_refuse_bad_arguments():
    from monoport_b200 import _lib
    from monoport_b200.modeling.MonoPortNet import FeatureHandle
    from monoport_b200.pipeline import FrameGraph
    from monoport_b200.recon import McubesWorkspace, marching_cubes_async
    lib = _lib.load()
    st = _lib.stream_ptr()
    netC = _colour_net()
    netG = build_net("G", *spec.make_weights(spec.G_CHANNELS, 3))
    buf = torch.zeros(4096, dtype=torch.int64, device="cuda")
    p = ctypes.c_void_p(buf.data_ptr())
    c12 = _lib.calib12(spec.scene_calib(20, 33))
    # mp_mcubes_run_async
    ws = McubesWorkspace((9, 9, 9), "cuda")
    vol = torch.zeros((9, 9, 9), device="cuda")
    vp = ctypes.c_void_p(vol.data_ptr())

    def mc(v_cap=16, f_cap=16, counts=p, c32=p, world=None, verts=p):
        return lib.mp_mcubes_run_async(ws.ptr, vp, ctypes.c_float(0.5), world, v_cap, f_cap, verts, p, counts, c32, st)
    assert mc() == _lib.MP_OK
    assert mc(v_cap=-1) == -1 and mc(f_cap=-1) == -1 and mc(v_cap=1 << 31) == -1
    assert mc(counts=None) == -1 and mc(c32=None) == -1 and mc(verts=None) == -1
    assert mc(v_cap=0, verts=None) == _lib.MP_OK
    assert mc(world=(ctypes.c_float * 7)(0.0, -1, -1, -1, 1, 1, 1)) == -1
    assert lib.mp_mcubes_run_async(None, vp, ctypes.c_float(0.5), None, 16, 16, p, p, p, p, st) == -1
    # mp_query_points_count / mp_mesh_normals_async
    fc = netC.feature_handle(spec.make_feat(512, 16, 16, 1).cuda())
    fg = netG.feature_handle(spec.make_feat(256, 16, 16, 1).cuda())
    fb = FeatureHandle(512, 16, 16, torch.device("cuda"), B=2)
    hc, hg = netC.surface_classifier.handle(), netG.surface_classifier.handle()

    def q(head, fh, n=8):
        return lib.mp_query_points_count(head, fh.ptr, p, n, 1, 3, c12, 0, ctypes.c_float(1.28), p, max(n, 0), p,
                                         _lib.MODE_AUTO, st)
    assert q(hc, fc) == _lib.MP_OK
    assert q(hc, fb) == -1 and q(hc, fc, n=-1) == -1

    def mn(head, fh, cap=8, counts=p):
        return lib.mp_mesh_normals_async(head, fh.ptr, p, counts, p, cap, c12, 0, ctypes.c_float(1.28), _lib.MODE_AUTO, p, p, st)
    assert mn(hg, fg) == _lib.MP_OK
    assert mn(hc, fc) == -1                              # a 3-output head
    assert mn(hg, fb) == -1 and mn(hg, fg, cap=-1) == -1 and mn(hg, fg, counts=None) == -1
    torch.cuda.synchronize()
    # the Python layer
    with pytest.raises(ValueError):
        marching_cubes_async(torch.zeros((9, 9, 10), device="cuda"), torch.empty((4, 3), device="cuda"),
                             torch.empty((4, 3), dtype=torch.int32, device="cuda"),
                             torch.empty(2, dtype=torch.int64, device="cuda"), torch.empty(1, dtype=torch.int32, device="cuda"),
                             workspace=ws)
    with pytest.raises(ValueError):
        marching_cubes_async(vol, torch.empty((4, 3), device="cuda"), torch.empty((4, 3), device="cuda"),
                             torch.empty(2, dtype=torch.int64, device="cuda"), torch.empty(1, dtype=torch.int32, device="cuda"),
                             workspace=ws)
    ws.close()
    net, _ = _person_frames()
    eng = _engine(net, True)
    cal = spec.scene_calib(20, 33)
    with pytest.raises(ValueError):
        FrameGraph(net, eng, cal, with_encoder=False, mesh_normals=True)
    with pytest.raises(ValueError):
        FrameGraph(net, eng, cal, with_encoder=False, mesh=True, mesh_colours=True)
    g = FrameGraph(net, eng, cal, with_encoder=False)
    with pytest.raises(RuntimeError):
        g.mesh()
    g.close()
    g = FrameGraph(net, eng, cal, with_encoder=False, mesh=True)
    with pytest.raises(RuntimeError):
        g.mesh()
    g.close()
