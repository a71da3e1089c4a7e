"""The mesh renderer on the GPU (mp_render_mesh_async, recon.render_mesh, FrameGraph(views=...); DESIGN.md §F3.2): the
kernels equal the numpy restatement tests/raster_ref.py bit for bit; a captured render equals the eager one; captured frames
equal the eager chain reconstruction -> mesh_normals / mesh_colours -> render_mesh; the normal image of a dense sphere
against its analytic normals; the coverage of an orthographic front view against forward_vertices' visible columns; and the
refusals.  (There is no OpenGL on these machines: parity with GL itself is not pinned.)"""
import ctypes

import numpy as np
import pytest
import torch

import raster_ref
import render_cases
from helpers import build_net
from oracle import spec

pytestmark = pytest.mark.gpu

B_MIN, B_MAX = (-1.0, -1.0, -1.0), (1.0, 1.0, 1.0)
B = np.array([[-1.0, -1.0, -1.0]], dtype=np.float32)
CAL = spec.scene_calib(20, 33)


def _person(n=3):
    Ws, bs = spec.make_weights(spec.G_CHANNELS, 3)
    base = spec.make_feat(256, 128, 128, 4, 0.5)
    feats = []
    for k in range(n):
        W2, b2, f, _ = spec.heightfield_person(Ws, bs, base * (1.0 + 0.1 * k), channel=0)
        feats.append(f.cuda())
    return build_net("G", W2, b2), feats


def _engine(net, res=(17, 33, 65)):
    from monoport_b200.engine import Seg3dLossless, make_query_func
    return Seg3dLossless(make_query_func(net), B, -B, list(res), balance_value=0.5, faster=True).to("cuda")


def _colour_net():
    Wc, bc = spec.make_weights(spec.C_CHANNELS, 21)
    return build_net("C", Wc, bc)


def _render_dev(c, normals=True, colours=True, clear=(0, 0, 0, 0)):
    """mp_render_mesh_async on a case's buffers and counts as they are"""
    from monoport_b200 import _lib
    from monoport_b200.recon import MeshRenderer
    d = {k: torch.from_numpy(np.ascontiguousarray(c[k])).cuda() for k in ("verts", "faces", "counts", "mats", "normals", "colours")}
    r = MeshRenderer(c["faces"].shape[0], c["mats"].shape[0], (c["W"], c["H"]), normals, colours, "cuda", clear)
    r.enqueue(d["verts"], d["faces"], d["counts"], d["normals"] if normals else None, d["colours"] if colours else None,
              d["mats"], _lib.stream_ptr(torch.device("cuda")))
    torch.cuda.synchronize()
    return (None if r.normal is None else r.normal.cpu().numpy(), None if r.colour is None else r.colour.cpu().numpy())


def same_bits(a, b):
    """equal bits, NaN at the same places (the device's and numpy's NaN payloads differ)"""
    if a is None or b is None:
        return a is None and b is None
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(a.view(np.uint32)[~na], b.view(np.uint32)[~nb])


@pytest.fixture(scope="module")
def all_cases(golden_dir):
    out = render_cases.cases(golden_dir)
    big = render_cases.cases(golden_dir, size=512)
    out["fv_two_blobs_65_ortho33_512"] = big["fv_two_blobs_65_ortho33"]
    out["persp_near_512"] = big["persp_near"]
    return out


@pytest.mark.parametrize("name", ["fv_sphere_33_ortho0", "fv_sphere_33_ortho33", "fv_two_blobs_65_ortho0",
                                  "fv_two_blobs_65_ortho33", "fv_corner_33_ortho0", "fv_corner_33_ortho33",
                                  "fv_noise_33_ortho0", "fv_noise_33_ortho33", "persp_near", "quad_large", "quad_guard",
                                  "quad_persp", "coincident", "degenerate", "beyond_count", "views3", "nonsquare_96x64",
                                  "fv_two_blobs_65_ortho33_512", "persp_near_512"])
def test_kernels_equal_the_restatement(all_cases, name):
    c = all_cases[name]
    got = _render_dev(c, clear=(0.25, 0.5, 0.75, 0.0))
    want = raster_ref.render(c["verts"], c["faces"], c["counts"], c["mats"], c["W"], c["H"], c["normals"], c["colours"],
                             clear=(0.25, 0.5, 0.75, 0.0))
    assert same_bits(got[0], want[0]) and same_bits(got[1], want[1])


def test_render_mesh_eager_and_one_attribute(all_cases):
    from monoport_b200.recon import render_mesh
    c = all_cases["views3"]
    M = torch.from_numpy(c["mats"][:, :16].reshape(-1, 4, 4).copy())
    P = c["mats"][:, 16:].reshape(-1, 4, 4).copy()                       # (numpy and torch matrices mix)
    v, f = torch.from_numpy(c["verts"]).cuda(), torch.from_numpy(c["faces"]).cuda()
    n, col = render_mesh(v, f, M, P, (c["W"], c["H"]), normals=torch.from_numpy(c["normals"]).cuda(),
                         colours=torch.from_numpy(c["colours"]).cuda())
    want = raster_ref.render(c["verts"], c["faces"], c["counts"], c["mats"], c["W"], c["H"], c["normals"], c["colours"])
    assert same_bits(n.cpu().numpy(), want[0]) and same_bits(col.cpu().numpy(), want[1])
    n1, col1 = render_mesh(v, f, M[0], P[0], (c["W"], c["H"]), colours=torch.from_numpy(c["colours"]).cuda())
    assert n1 is None and col1.shape == (1, c["H"], c["W"], 4) and torch.equal(col1[0], col[0])


def test_captured_render_equals_eager(all_cases):
    from monoport_b200 import _lib
    from monoport_b200.recon import MeshRenderer, render_mesh, view_mats
    c = all_cases["persp_near"]
    v, f = torch.from_numpy(c["verts"]).cuda(), torch.from_numpy(c["faces"]).cuda()
    nrm, col = torch.from_numpy(c["normals"]).cuda(), torch.from_numpy(c["colours"]).cuda()
    counts = torch.tensor([v.shape[0], f.shape[0]], dtype=torch.int64, device="cuda")
    M, P = c["mats"][0, :16].reshape(4, 4), c["mats"][0, 16:].reshape(4, 4)
    mats = view_mats(M, P, "cuda")
    r = MeshRenderer(f.shape[0], 1, (c["W"], c["H"]), True, True, "cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        r.enqueue(v, f, counts, nrm, col, mats, _lib.stream_ptr(torch.device("cuda")))
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        r.enqueue(v, f, counts, nrm, col, mats, _lib.stream_ptr(torch.device("cuda")))
    for pitch in (20, -40):                                                  # the graph follows the views written before a replay
        M2 = render_cases.model(pitch, 30, (0.1, 0.0, -0.35))
        mats.copy_(view_mats(M2, P, "cuda"))
        r.normal.fill_(-1)
        g.replay()
        torch.cuda.synchronize()
        en, ec = render_mesh(v, f, M2, P, (c["W"], c["H"]), normals=nrm, colours=col)
        assert same_bits(r.normal.cpu().numpy(), en.cpu().numpy()) and torch.equal(r.colour, ec)


@pytest.mark.parametrize("n_lanes", [1, 2])
def test_captured_frames_equal_the_eager_chain(n_lanes):
    """Frames with their own cameras and views: the person, an empty frame, the person from another camera and other views.
    V = 2.  Each equals reconstruction(refine=2) -> mesh_normals("auto") / mesh_colours -> render_mesh bit for bit, and every
    other output equals a graph's without views."""
    from monoport_b200.pipeline import FrameGraph, FrameGraphRing
    from monoport_b200.recon import mesh_colours, mesh_normals, reconstruction, render_mesh
    net, feats = _person()
    netC = _colour_net()
    eng = _engine(net)
    c0 = spec.make_feat(512, 128, 128, 22, 0.5).cuda()
    empty = feats[0].clone()
    empty[0, 0] = -5.0
    frames = [(feats[0], c0), (empty, c0), (feats[2], c0), (feats[1], c0)]
    cams = [spec.scene_calib(20, 33), spec.scene_calib(20, 33), spec.scene_calib(20, 90), spec.scene_calib(20, 9)]
    O, Pp = render_cases.demo_ortho(), render_cases.perspective(60, 96 / 80, 0.5, 5.0)
    default = (np.stack([render_cases.model(0), render_cases.model(33, 20)]), np.stack([O, Pp]))
    other = (np.stack([render_cases.model(-10, 90), render_cases.model(0, 0, (0.1, 0.0, -0.3))]),
             np.stack([O, render_cases.perspective(90, 96 / 80)]))
    views = [None, None, other, None]
    size = (96, 80)
    want = []
    for (f, c), cam, vw in zip(frames, cams, views):
        r = reconstruction(net, "cuda", cam.cuda(), 65, B_MIN, B_MAX, use_octree=True, feats=[[f]], engine=eng, refine=2)
        if isinstance(r, int):
            want.append(None)
            continue
        verts, faces, _, _ = r
        nrm = mesh_normals(net, [[f]], verts, cam.cuda(), precision="auto")
        col = mesh_colours(netC, [[c]], verts, cam.cuda())
        vw = vw or default
        want.append(render_mesh(verts, faces, vw[0], vw[1], size, normals=nrm, colours=col))
    assert want[1] is None and want[0] is not None
    plain = FrameGraphRing(lambda: FrameGraph(net, eng, CAL, "front", with_encoder=False, netC=netC, mesh=True,
                                              mesh_normals=True, mesh_colours=True, mesh_refine=2), n_lanes=n_lanes)
    base = [tuple(None if t is None else t.clone() for t in out) for out in plain.run(iter(frames), calibs=cams)]
    plain.close()
    ring = FrameGraphRing(lambda: FrameGraph(net, eng, CAL, "front", with_encoder=False, netC=netC, mesh=True,
                                             mesh_normals=True, mesh_colours=True, mesh_refine=2, views=default,
                                             view_size=size), n_lanes=n_lanes)
    for i, (w, b, out) in enumerate(zip(want, base, ring.run(iter(frames), calibs=cams, views=views))):
        assert len(out) == len(b) + 2
        for k in range(len(b)):
            assert (b[k] is None and out[k] is None) or torch.equal(b[k], out[k]), (i, k)
        n, col = out[-2:]
        assert n.shape == (2, 80, 96, 4) and col.shape == (2, 80, 96, 4)
        if w is None:
            assert (n == 0).all() and (col == 0).all()
            continue
        assert same_bits(n.cpu().numpy(), w[0].cpu().numpy()), i
        assert torch.equal(col, w[1]), i
        assert (n[..., 3] == 1).any()
    ring.close()


def test_frame_without_views_is_unchanged_and_overflow_raises():
    from monoport_b200.pipeline import FrameGraph
    net, feats = _person(1)
    eng = _engine(net)
    views = (render_cases.model(0), render_cases.demo_ortho())
    fg = FrameGraph(net, eng, CAL, "front", with_encoder=False, mesh=True, mesh_normals=True, mesh_capacity=(100, 100),
                    views=views, view_size=(32, 32))
    fg.launch(feats[0])
    fg.result()
    with pytest.raises(RuntimeError, match="capacity"):
        fg.mesh_rendered()
    fg.close()
    with pytest.raises(RuntimeError, match="views="):
        g = FrameGraph(net, eng, CAL, "front", with_encoder=False, mesh=True, mesh_normals=True)
        g.launch(feats[0])
        g.result()
        g.mesh_rendered()
    with pytest.raises(ValueError, match="views needs"):
        FrameGraph(net, eng, CAL, "front", with_encoder=False, mesh=True, views=views, view_size=(8, 8))
    with pytest.raises(ValueError, match="view_size"):
        FrameGraph(net, eng, CAL, "front", with_encoder=False, mesh=True, mesh_normals=True, views=views)


def test_sphere_normals_against_the_analytic_normals():
    """a dense marching-cubes sphere (R = 129, radius 0.6) with exact unit vertex normals, drawn orthographically from the
    front at 256 x 256: away from the silhouette (|xy| < 0.9 r) every pixel's normal colour is within 1e-3 of the analytic
    normal's at the sphere point the pixel sees"""
    from monoport_b200.recon import marching_cubes, render_mesh
    R, r0 = 129, 0.6
    g = (torch.arange(R, dtype=torch.float32, device="cuda") + 0.5) * (2.0 / R) - 1.0
    z, y, x = torch.meshgrid(g, g, g, indexing="ij")
    vol = torch.sigmoid(20.0 * (r0 - torch.sqrt(x * x + y * y + z * z))).contiguous()
    v, f = marching_cubes(vol, 0.5)
    v = (v + 0.5) * (2.0 / R) - 1.0
    n = v / v.norm(dim=1, keepdim=True)
    S = 256
    img, _ = render_mesh(v, f, render_cases.model(0), render_cases.demo_ortho(), (S, S), normals=n)
    img = img[0].cpu().numpy()
    c = (np.arange(S) + 0.5) * (2.0 / S) - 1.0
    X, Y = np.meshgrid(c, c[::-1], indexing="xy")                             # row 0 is the top
    rho2 = X * X + Y * Y
    inner = rho2 < (0.9 * r0) ** 2
    Z = np.sqrt(np.maximum(r0 * r0 - rho2, 0))
    want = (np.stack([X, Y, Z], -1) / r0 + 1) / 2
    assert (img[..., 3][inner] == 1).all()
    err = np.abs(img[..., :3] - want)[inner].max()
    assert err < 1e-3, err


def test_front_view_coverage_agrees_with_visible_columns():
    """an orthographic front view at R x R whose pixel centres sit on the grid's (x, y) nodes covers the columns
    forward_vertices finds visible on >= 99 % of the pixels on the person"""
    from monoport_b200.recon import forward_vertices, marching_cubes, render_mesh
    net, feats = _person(1)
    R = 129
    sdf = _engine(net, (17, 33, 65, 129))(im_feat_list=[[feats[0]]], calib_tensor=CAL.cuda())
    X, Y, _, _ = forward_vertices(sdf, "front")
    v, f = marching_cubes(sdf[0, 0].contiguous(), 0.5)                      # index space: (x, y, z)
    M = np.diag([2.0 / R, 2.0 / R, 1.0 / R, 1.0])
    M[:3, 3] = (1.0 / R - 1, 1.0 / R - 1, -0.5)                             # pixel centre i + 1/2 <-> node x = i
    _, col = render_mesh(v, f, M, np.eye(4), (R, R), colours=torch.ones_like(v))
    covered = (col[0, ..., 3] == 1).cpu().numpy()[::-1]                       # [y][x], y from the bottom
    visible = np.zeros((R, R), dtype=bool)
    visible[Y.cpu().numpy(), X.cpu().numpy()] = True
    person = covered | visible
    assert person.sum() > 500
    agree = (covered == visible)[person].mean()
    assert agree >= 0.99, agree


def test_refusals():
    from monoport_b200 import _lib
    from monoport_b200.recon import render_mesh
    lib = _lib.load()
    buf = torch.zeros(1 << 20, dtype=torch.float32, device="cuda")
    p = ctypes.c_void_p(buf.data_ptr())
    clear = (ctypes.c_float * 4)(0, 0, 0, 0)
    st = _lib.stream_ptr(torch.device("cuda"))

    def call(verts=p, faces=p, counts=p, v_cap=8, f_cap=8, nrm=p, col=p, mats=p, V=1, W=16, H=16, clr=clear, on=p, oc=p,
             scratch=p):
        return lib.mp_render_mesh_async(verts, faces, counts, v_cap, f_cap, nrm, col, mats, V, W, H, clr, on, oc, scratch, st)

    assert call() == _lib.MP_OK
    torch.cuda.synchronize()
    bad = [dict(verts=None), dict(faces=None), dict(counts=None), dict(mats=None), dict(scratch=None), dict(clr=None),
           dict(nrm=None, col=None, on=None, oc=None), dict(nrm=None), dict(col=None), dict(on=None), dict(oc=None),
           dict(V=0), dict(V=-1), dict(W=0), dict(H=0), dict(W=8193), dict(H=8193), dict(v_cap=-1), dict(f_cap=-1),
           dict(v_cap=1 << 31), dict(f_cap=1 << 31)]
    for kw in bad:
        assert call(**kw) != _lib.MP_OK, kw
        assert lib.mp_last_error(), kw
    assert call(verts=None, v_cap=0) == _lib.MP_OK and call(faces=None, f_cap=0) == _lib.MP_OK
    assert lib.mp_render_mesh_scratch_bytes(8, 0, 16, 16) == -1 and lib.mp_render_mesh_scratch_bytes(-1, 1, 16, 16) == -1
    assert lib.mp_render_mesh_scratch_bytes(8, 1, 8193, 16) == -1
    torch.cuda.synchronize()
    v = torch.zeros((3, 3), device="cuda")
    f = torch.zeros((1, 3), dtype=torch.int32, device="cuda")
    with pytest.raises(ValueError):
        render_mesh(v, f, np.eye(4), np.eye(4), (16, 16))
    with pytest.raises(ValueError):
        render_mesh(v, f, np.eye(3), np.eye(4), (16, 16), normals=v)
    with pytest.raises(ValueError):
        render_mesh(v, f, np.eye(4), np.eye(4), (0, 16), normals=v)
    with pytest.raises(ValueError):
        render_mesh(v, f, np.stack([np.eye(4)] * 2), np.stack([np.eye(4)] * 3), (16, 16), normals=v)
