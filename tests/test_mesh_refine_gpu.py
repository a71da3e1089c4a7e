"""The mesh refinement on the GPU (refine_mesh_async / mp_mesh_refine_async, reconstruction(refine=K), FrameGraph(mesh_refine=K);
DESIGN.md §F3.1): K = 0 and K = 1 change nothing; the kernels equal the float32 restatement (tests/mesh_refine_ref.py) driven by
net.query bit for bit, over precisions, cameras, volumes and heads; every refined vertex stays on its edge and is no further
from the iso level than the marching-cubes vertex; the accuracy against a float64 evaluation of the head; the captured frame
equals the eager chain; and the refusals of the new entry points."""
import ctypes

import numpy as np
import pytest
import torch

from helpers import build_net
from mesh_refine_ref import mc_edges, query64, refine_mesh_ref
from oracle import spec

pytestmark = pytest.mark.gpu

B_MIN, B_MAX = (-1.0, -1.0, -1.0), (1.0, 1.0, 1.0)
B = np.array([[-1.0, -1.0, -1.0]], dtype=np.float32)
CAL = spec.scene_calib(20, 33)


def _person(proj="orthogonal", n=3):
    Ws, bs = spec.make_weights(spec.G_CHANNELS, 3)
    base = spec.make_feat(256, 128, 128, 4, 0.5)
    feats = []
    for k in range(n):
        W2, b2, f, _ = spec.heightfield_person(Ws, bs, base * (1.0 + 0.1 * k), channel=0)
        feats.append(f.cuda())
    return build_net("G", W2, b2, proj=proj), feats, (W2, b2)


def _random(proj="orthogonal"):
    Ws, bs = spec.make_weights(spec.G_CHANNELS, 3)
    return build_net("G", Ws, bs, proj=proj), [spec.make_feat(256, 128, 128, 4).cuda()], (Ws, bs)


def _engine(net, faster, res=(17, 33, 65)):
    from monoport_b200.engine import Seg3dLossless, make_query_func
    return Seg3dLossless(make_query_func(net), B, -B, list(res), balance_value=0.5, faster=faster).to("cuda")


def _colour_net():
    Wc, bc = spec.make_weights(spec.C_CHANNELS, 21)
    return build_net("C", Wc, bc)


def _volume(net, feat, cal, source):
    if source == "lossless65":
        return _engine(net, False)(im_feat_list=[[feat]], calib_tensor=cal)[0, 0].clone()
    R = 33 if source == "dense33" else 65
    return net.query_grid(feat, cal, R, torch.tensor(B_MIN), torch.tensor(B_MAX))


def _refined(net, feat, vol, cal, rounds, guard=0):
    """marching_cubes_async (world) + refine_mesh_async on one workspace -> (MC verts, refined verts, faces, guard rows)"""
    from monoport_b200.recon import McubesWorkspace, marching_cubes_async, refine_mesh_async
    R = vol.shape[-1]
    ws = McubesWorkspace(vol.shape, "cuda")
    cap = 3 * R ** 3
    vb = torch.full((cap + guard, 3), -12345.0, device="cuda")
    fb = torch.empty((6 * cap, 3), dtype=torch.int32, device="cuda")
    counts = torch.zeros(2, dtype=torch.int64, device="cuda")
    c32 = torch.zeros(1, dtype=torch.int32, device="cuda")
    marching_cubes_async(vol, vb[:cap], fb, counts, c32, 0.5, B_MIN, B_MAX, workspace=ws)
    torch.cuda.synchronize()
    nv, nf = counts.tolist()
    mc = vb[:nv].clone()
    refine_mesh_async(net, feat, vol, vb[:cap], c32, rounds, B_MIN, B_MAX, cal, workspace=ws)
    torch.cuda.synchronize()
    ws.close()
    return mc, vb[:nv].clone(), fb[:nf].clone(), vb[nv:]


def _query(net, feat, cal):
    def fn(p):
        return net.query([[feat]], p.cuda()[None], cal)[0][0, 0]
    return fn


@pytest.mark.parametrize("K", [0, 1])
def test_zero_and_one_round_change_nothing(K):
    from monoport_b200.pipeline import FrameGraph
    from monoport_b200.recon import reconstruction
    net, feats, _ = _person()
    cal = CAL.cuda()
    eng = _engine(net, True)
    for f in feats[:2]:
        want = reconstruction(net, "cuda", cal, 65, B_MIN, B_MAX, use_octree=True, feats=[[f]], engine=eng)
        got = reconstruction(net, "cuda", cal, 65, B_MIN, B_MAX, use_octree=True, feats=[[f]], engine=eng, refine=K)
        assert torch.equal(want[0], got[0]) and torch.equal(want[1], got[1])
        dense = reconstruction(net, "cuda", cal, 33, B_MIN, B_MAX, feats=[[f]])
        got = reconstruction(net, "cuda", cal, 33, B_MIN, B_MAX, feats=[[f]], refine=K)
        assert torch.equal(dense[0], got[0]) and torch.equal(dense[1], got[1])
    plain = FrameGraph(net, eng, CAL, "front", with_encoder=False, mesh=True)
    ref = FrameGraph(net, eng, CAL, "front", with_encoder=False, mesh=True, mesh_refine=K)
    for f in feats:
        plain.launch(f).result()
        a = [t.clone() for t in plain.mesh()[:2]]
        ref.launch(f).result()
        b = ref.mesh()[:2]
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    plain.close()
    ref.close()


# (under the perspective camera the person is small in the image: the lossless engine's 17^3 level finds no surface and the
# frame is empty -- the dense 65^3 volume has a few hundred vertices -- so that case has nothing to refine)
CASES = [(prec, cam, src, head) for prec in ("fp32", "tc") for cam in ("rot", "persp", "none")
         for src in ("dense33", "dense65", "lossless65") for head in ("random", "person")
         if (cam, src, head) != ("persp", "lossless65", "person")]


@pytest.mark.parametrize("prec,cam,src,head", CASES)
def test_kernels_equal_the_restatement_and_keep_the_invariants(prec, cam, src, head):
    proj = "perspective" if cam == "persp" else "orthogonal"
    net, feats, _ = (_random if head == "random" else _person)(proj)
    net.precision = prec
    feat = feats[0]
    cal = None if cam == "none" else CAL.cuda()
    if src == "lossless65" and cal is None:
        cal = torch.eye(4)[None].cuda()                       # (the engine needs a camera: the identity is calibs=None's mapping)
    vol = _volume(net, feat, cal, src)
    K = 4
    mc, got, faces, _ = _refined(net, feat, vol, cal, K)
    assert mc.shape[0] > 0 or cam == "persp", "no surface"
    want, want_faces = refine_mesh_ref(_query(net, feat, cal), vol, 0.5, K, B_MIN, B_MAX)
    assert torch.equal(faces.cpu(), want_faces)
    assert torch.equal(got.cpu(), want), "differs from the restatement at %d of %d vertices" % (
        int((got.cpu() != want).any(1).sum()), want.shape[0])
    # invariants: on the edge, between its end points, and no further from iso than the marching-cubes vertex
    xx, yy, zz, aa = mc_edges(vol.cpu().numpy())
    a = torch.as_tensor(aa).cuda()
    idx = torch.arange(len(aa), device="cuda")
    keep = torch.ones_like(mc, dtype=torch.bool)
    keep[idx, a] = False
    assert torch.equal(got[keep], mc[keep])
    R = vol.shape[-1]
    scale = (torch.tensor(B_MAX) - torch.tensor(B_MIN)) / R
    base = torch.stack([torch.as_tensor(xx), torch.as_tensor(yy), torch.as_tensor(zz)], 1).float().cuda()
    lo = ((base + 0.5) * scale.cuda() + torch.tensor(B_MIN).cuda())[idx, a]
    hi = ((base + 1.5) * scale.cuda() + torch.tensor(B_MIN).cuda())[idx, a]
    assert bool(((got[idx, a] >= lo) & (got[idx, a] <= hi)).all())
    q = _query(net, feat, cal)
    e_mc, e_got = (q(mc.t()) - 0.5).abs(), (q(got.t()) - 0.5).abs()
    assert bool((e_got <= e_mc).all())
    print("%s %s %s %s: %d vertices, max |sigma - iso| MC %.3e, refined (K=%d) %.3e"
          % (prec, cam, src, head, mc.shape[0], e_mc.max().item(), K, e_got.max().item()))


@pytest.mark.parametrize("prec,bar", [("fp32", 1e-4), ("tc", 2e-4)])
def test_accuracy_against_float64(prec, bar):
    """K = 8 on the person's dense 65^3 volume: p99 of |sigma64(v) - iso| over the vertices whose float64 end values bracket
    iso, against the marching-cubes vertices' figure"""
    net, feats, (Ws, bs) = _person()
    net.precision = prec
    feat, cal = feats[0], CAL.cuda()
    vol = _volume(net, feat, cal, "dense65")
    mc, got, _, _ = _refined(net, feat, vol, cal, 8)
    xx, yy, zz, aa = mc_edges(vol.cpu().numpy())

    def s64(p):
        return query64(feat, p, cal, [w.cuda() for w in Ws], [b.cuda() for b in bs])[0]
    base = torch.stack([torch.as_tensor(xx), torch.as_tensor(yy), torch.as_tensor(zz)], 1).double().cuda()
    idx, a = torch.arange(len(aa), device="cuda"), torch.as_tensor(aa).cuda()
    ends = []
    for k in (0, 1):
        p = base.clone()
        p[idx, a] += k
        ends.append(s64(((p + 0.5) * (2.0 / 65) - 1.0).t()) - 0.5)
    bracket = (ends[0] > 0) != (ends[1] > 0)
    e_mc = (s64(mc.double().t()) - 0.5).abs()[bracket]
    e_got = (s64(got.double().t()) - 0.5).abs()[bracket]
    qs = torch.tensor([0.5, 0.99], dtype=torch.float64, device="cuda")
    m, g = torch.quantile(e_mc, qs).tolist(), torch.quantile(e_got, qs).tolist()
    print("%s, R=65, %d of %d vertices bracketed: |sigma64 - iso| MC p50 %.3e p99 %.3e max %.3e; refined (K=8) p50 %.3e "
          "p99 %.3e max %.3e" % (prec, int(bracket.sum()), len(aa), m[0], m[1], e_mc.max().item(), g[0], g[1], e_got.max().item()))
    assert int(bracket.sum()) > 0.9 * len(aa)
    assert g[1] <= bar


def test_no_vertex_beyond_the_count_is_written():
    from monoport_b200.recon import McubesWorkspace, marching_cubes, marching_cubes_async, refine_mesh_async
    net, feats, _ = _person()
    feat, cal = feats[0], CAL.cuda()
    vol = _volume(net, feat, cal, "dense33")
    V, _ = marching_cubes(vol)
    ws = McubesWorkspace(vol.shape, "cuda")
    for vc in (V.shape[0] - 9, 0):
        vb = torch.full((vc + 64, 3), -12345.0, device="cuda")
        fb = torch.empty((4 * V.shape[0], 3), dtype=torch.int32, device="cuda")
        counts = torch.zeros(2, dtype=torch.int64, device="cuda")
        c32 = torch.zeros(1, dtype=torch.int32, device="cuda")
        marching_cubes_async(vol, vb[:vc], fb, counts, c32, 0.5, B_MIN, B_MAX, workspace=ws)
        refine_mesh_async(net, feat, vol, vb[:vc], c32, 3, B_MIN, B_MAX, cal, workspace=ws)
        torch.cuda.synchronize()
        assert c32.item() == vc and bool((vb[vc:] == -12345.0).all())
    ws.close()


@pytest.mark.parametrize("n_lanes", [1, 2])
def test_captured_frames_equal_the_eager_chain(n_lanes):
    """Frames with their own cameras (launch(calib=...)): the person, a ridge, an empty frame, the person from another view.
    mesh_refine=4 with normals and colours equals reconstruction(refine=4) -> mesh_normals("auto") -> mesh_colours at the
    refined vertices, bit for bit; every other output equals a graph's without the refinement."""
    from monoport_b200.pipeline import FrameGraph, FrameGraphRing
    from monoport_b200.recon import mesh_colours, mesh_normals, reconstruction
    net, feats, _ = _person()
    netC = _colour_net()
    eng = _engine(net, True)
    c0 = spec.make_feat(512, 128, 128, 22, 0.5).cuda()
    empty = feats[0].clone()
    empty[0, 0] = -5.0
    ridge = feats[1].clone()
    d = torch.arange(4, 60, device=ridge.device)
    ridge[0, 0, d, d] = 0.3
    frames = [(feats[0], c0), (ridge, c0), (empty, c0), (feats[2], c0)]
    cams = [spec.scene_calib(20, 33), spec.scene_calib(20, 9), spec.scene_calib(20, 33), spec.scene_calib(20, 90)]
    want = []
    for (f, c), cam in zip(frames, cams):
        r = reconstruction(net, "cuda", cam.cuda(), 65, B_MIN, B_MAX, use_octree=True, feats=[[f]], engine=eng, refine=4,
                           normals=True)
        if isinstance(r, int):
            want.append(None)
            continue
        verts, faces, nrm, _ = r
        exact = mesh_normals(net, [[f]], verts, cam.cuda(), precision="fp32")
        assert (exact - nrm).abs().max().item() <= 1e-6
        want.append((verts, faces, mesh_normals(net, [[f]], verts, cam.cuda(), precision="auto"),
                     mesh_colours(netC, [[c]], verts, cam.cuda())))
    assert want[2] is None and want[0] is not None
    plain = FrameGraphRing(lambda: FrameGraph(net, eng, CAL, "front", with_encoder=False, netC=netC, mesh=True),
                           n_lanes=n_lanes)
    base = [tuple(None if t is None else t.clone() for t in out) for out in plain.run(iter(frames), calibs=cams)]
    plain.close()
    ring = FrameGraphRing(lambda: FrameGraph(net, eng, CAL, "front", with_encoder=False, netC=netC, mesh=True,
                                             mesh_normals=True, mesh_colours=True, mesh_refine=4), n_lanes=n_lanes)
    for i, (w, b, out) in enumerate(zip(want, base, ring.run(iter(frames), calibs=cams))):
        assert len(out) == 11
        for k in range(7):
            assert (b[k] is None and out[k] is None) or torch.equal(b[k], out[k]), (i, k)
        if w is None:
            assert all(t is None for t in out[7:])
            continue
        assert torch.equal(b[8], out[8])                                         # faces: marching cubes'
        for name, x, y in zip(("verts", "faces", "normals", "colours"), w, out[7:]):
            assert x.shape == y.shape and torch.equal(x, y), (i, name)
    ring.close()


def test_overflowing_frame_still_raises():
    from monoport_b200.pipeline import FrameGraph
    from monoport_b200.recon import marching_cubes
    net, feats, _ = _person()
    eng = _engine(net, True)
    vol = eng(im_feat_list=[[feats[0]]], calib_tensor=CAL.cuda())[0, 0].clone()
    V, F = marching_cubes(vol)
    fg = FrameGraph(net, eng, CAL, "front", with_encoder=False, mesh=True, mesh_capacity=(V.shape[0] - 1, F.shape[0]),
                    mesh_refine=3)
    assert fg.launch(feats[0]).result()[0] is not None
    with pytest.raises(RuntimeError, match="reconstruction"):
        fg.mesh()
    fg.close()


def test_refusals():
    from monoport_b200 import _lib
    from monoport_b200.modeling.MonoPortNet import FeatureHandle
    from monoport_b200.pipeline import FrameGraph
    from monoport_b200.recon import McubesWorkspace, reconstruction, refine_mesh_async
    lib = _lib.load()
    st = _lib.stream_ptr()
    netC = _colour_net()
    netG = build_net("G", *spec.make_weights(spec.G_CHANNELS, 3))
    buf = torch.zeros(1 << 16, dtype=torch.int64, device="cuda")
    p = ctypes.c_void_p(buf.data_ptr())
    c12 = _lib.calib12(CAL)
    ws = McubesWorkspace((9, 9, 9), "cuda")
    vol = torch.zeros((9, 9, 9), device="cuda")
    vp = ctypes.c_void_p(vol.data_ptr())
    fc = netC.feature_handle(spec.make_feat(512, 16, 16, 1).cuda())
    fg = netG.feature_handle(spec.make_feat(256, 16, 16, 1).cuda())
    fb = FeatureHandle(256, 16, 16, torch.device("cuda"), B=2)
    hc, hg = netC.surface_classifier.handle(), netG.surface_classifier.handle()
    w9 = (ctypes.c_float * 7)(9.0, -1, -1, -1, 1, 1, 1)

    def rf(head=hg, fh=fg, wsp=ws.ptr, vol_=vp, world=w9, verts=p, c32=p, v_cap=16, rounds=2, scratch=p):
        rc = lib.mp_mesh_refine_async(head, fh.ptr, wsp, vol_, ctypes.c_float(0.5), world, verts, c32, v_cap, rounds, c12, 0,
                                      ctypes.c_float(1.28), _lib.MODE_AUTO, scratch, st)
        return rc, lib.mp_last_error().decode()
    assert rf()[1].find("has not run marching cubes") >= 0          # (nothing to refine on a fresh workspace)
    assert lib.mp_mcubes_run_async(ws.ptr, vp, ctypes.c_float(0.5), None, 16, 16, p, p, p, p, st) == _lib.MP_OK
    assert rf()[0] == _lib.MP_OK
    for kw, msg in [(dict(wsp=None), "NULL argument"), (dict(vol_=None), "NULL argument"), (dict(world=None), "NULL argument"),
                    (dict(c32=None), "NULL argument"), (dict(verts=None), "NULL argument"), (dict(scratch=None), "NULL argument"),
                    (dict(rounds=-1), "bad rounds"), (dict(v_cap=-1), "bad capacity"), (dict(v_cap=1 << 31), "bad capacity"),
                    (dict(head=hc, fh=fc), "mesh refinement needs a head with one output"),
                    (dict(fh=fb), "single-map feature handle"),
                    (dict(world=(ctypes.c_float * 7)(17.0, -1, -1, -1, 1, 1, 1)), "not the side of the workspace")]:
        rc, err = rf(**kw)
        assert rc != _lib.MP_OK and msg in err, (kw, err)
    assert rf(verts=None, scratch=None, v_cap=0)[0] == _lib.MP_OK
    assert lib.mp_mesh_refine_async_dcal(hg, fg.ptr, ws.ptr, vp, ctypes.c_float(0.5), w9, p, p, 16, 2, None, 0,
                                         ctypes.c_float(1.28), _lib.MODE_AUTO, p, st) != _lib.MP_OK
    assert lib.mp_mesh_refine_scratch_bytes(-1) == -1 and lib.mp_mesh_refine_scratch_bytes(1000) >= 49 * 1000
    torch.cuda.synchronize()
    # the Python layer
    verts = torch.zeros((16, 3), device="cuda")
    c32 = torch.zeros(1, dtype=torch.int32, device="cuda")
    feat = spec.make_feat(256, 16, 16, 1).cuda()
    with pytest.raises(ValueError, match="workspace must be an open McubesWorkspace"):
        refine_mesh_async(netG, feat, torch.zeros((11, 11, 11), device="cuda"), verts, c32, 2, B_MIN, B_MAX, CAL, workspace=ws)
    with pytest.raises(ValueError, match="rounds must be an integer >= 0"):
        refine_mesh_async(netG, feat, vol, verts, c32, -1, B_MIN, B_MAX, CAL, workspace=ws)
    with pytest.raises(RuntimeError, match="mesh refinement needs a head with one output"):
        refine_mesh_async(netC, spec.make_feat(512, 16, 16, 1).cuda(), vol, verts, c32, 2, B_MIN, B_MAX, CAL, workspace=ws)
    ws.close()
    net, feats, _ = _person()
    with pytest.raises(ValueError, match="refine must be an integer >= 0"):
        reconstruction(net, "cuda", CAL.cuda(), 33, B_MIN, B_MAX, feats=[[feats[0]]], refine=-2)
    eng = _engine(net, True)
    with pytest.raises(ValueError, match="mesh_refine needs mesh=True"):
        FrameGraph(net, eng, CAL, with_encoder=False, mesh_refine=2)
    with pytest.raises(ValueError, match="mesh_refine must be an integer >= 0"):
        FrameGraph(net, eng, CAL, with_encoder=False, mesh=True, mesh_refine=-1)
