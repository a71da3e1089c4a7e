"""The reconstruction chain away from the demo's defaults: a box other than [-1,1]^3 (asymmetric, no power-of-two extent, cutting
the synthetic person), surfaces whose visible vertices have NaN depths, the top-k engine on the fused and captured paths
(including an empty frame), and a perspective projection through the lossless engine.  Each path is compared with the eager
chain or the Python-callback engine bit for bit, and with the fp32/fp64 restatements where the numbers are approximate."""
import numpy as np
import pytest
import torch

from oracle import spec
from grad_cases import query_grad_ref
from helpers import build_net

pytestmark = pytest.mark.gpu

B1 = ((-0.83, -1.17, -0.61), (0.91, 1.06, 0.77))
RES = [17, 33, 65]


def _box():
    return np.array([B1[0]], dtype=np.float32), np.array([B1[1]], dtype=np.float32)


def _person():
    Ws, bs = spec.make_weights(spec.G_CHANNELS, 3)
    base = spec.make_feat(256, 128, 128, 4, 0.5)
    feats = []
    for k in range(2):
        W2, b2, f, _ = spec.heightfield_person(Ws, bs, base * (1.0 + 0.1 * k), channel=0)
        feats.append(f.cuda())
    empty = feats[0].clone()
    empty[0, 0] = -5.0                                   # height map far below every node: nothing occupied
    return build_net("G", W2, b2), feats, empty, W2, b2


def _plain(net):
    def query(points, im_feat_list, calib_tensor):        # RTL/main.py:168-183 without the fused tag
        return net.query(im_feat_list, points=points.permute(0, 2, 1), calibs=calib_tensor)[0]
    return query


def _same(a, b):
    """bit-equal, NaN where the other is NaN"""
    if a is None or b is None:
        return a is None and b is None
    return a.shape == b.shape and bool(((a == b) | (torch.isnan(a) & torch.isnan(b))).all())


@pytest.mark.parametrize("mode", ["fp32", "tc"])
def test_topk_fused_equals_generic_including_an_empty_frame(mode):
    """Seg3dTopk(make_query_func(net)) runs the pyramid on the device; the callback engine steps it from Python.  Same volume
    and per-level counts, with a level of k = 0 and one whose k exceeds its res^3 -- and on a frame that is empty after level
    0, where both report [r0^3, 0, ...] and evaluate nothing more."""
    from monoport_b200.engine import Seg3dTopk, make_query_func
    net, feats, empty, _, _ = _person()
    if mode == "tc" and not net.surface_classifier.tc_supported():
        pytest.skip("no tensor-core program for this head")
    net.precision = mode
    cal = spec.scene_calib(20, 33).cuda()
    res, kpts = [17, 33, 65, 129], [0, 40000, 0, 150000]          # 40000 > 33^3
    fused = Seg3dTopk(make_query_func(net), *_box(), res, kpts).to("cuda")
    generic = Seg3dTopk(_plain(net), *_box(), res, kpts).to("cuda")
    for f in (feats[0], empty, feats[1]):
        a = fused(im_feat_list=[[f]], calib_tensor=cal)
        g = generic(im_feat_list=[[f]], calib_tensor=cal)
        assert fused.last_stats == generic.last_stats, (fused.last_stats, generic.last_stats)
        if g is None:
            assert a is None and generic.last_stats == [17 ** 3, 0, 0, 0]
        else:
            assert generic.last_stats == [17 ** 3, 33 ** 3, 0, 150000]
            assert a is not None and torch.equal(a, g)


def test_lossless_fused_perspective_equals_generic_and_oracle():
    """net.projection = perspective through the lossless engine over the box: the fused on-device pyramid (a graph with the
    conflict loop on the device) equals the callback engine bit for bit, and its fp32 mask is the oracle engine's driven by
    the restated perspective query, up to fp32 summation-order ties."""
    from monoport_b200.engine import Seg3dLossless, make_query_func
    from monoport_b200.modeling.geometry import perspective
    net, feats, _, Ws, bs = _person()
    net.projection = perspective
    net.precision = "fp32"
    cal = torch.diag(torch.tensor([0.25, 0.25, 0.5, 1.0]))[None].contiguous()
    cal[0, 2, 3] = 0.0123                               # depth 0.5 z + 0.0123: no node sits at depth 0
    feat = feats[0].cpu()

    def q(p):
        return spec.query_ref(feat, p.t().contiguous(), cal, Ws, bs, spec.LAST_SIGMOID, "perspective")[0]
    for balance in (0.5, 0.3):                          # (the conflict detection of the fused scatter uses the balance)
        fused = Seg3dLossless(make_query_func(net), *_box(), RES, balance_value=balance, faster=False).to("cuda")
        generic = Seg3dLossless(_plain(net), *_box(), RES, balance_value=balance, faster=False).to("cuda")
        a = fused(im_feat_list=[[feats[0]]], calib_tensor=cal.cuda())
        g = generic(im_feat_list=[[feats[0]]], calib_tensor=cal.cuda())
        assert a is not None and g is not None
        assert fused.last_stats == generic.last_stats and torch.equal(a, g), (balance, fused.last_stats, generic.last_stats)
        want = spec.seg3d_lossless_ref(q, RES, *B1, balance=balance, faster=False)
        assert want is not None and int((want > balance).sum()) > 100
        assert ((a[0, 0].cpu() > balance) != (want > balance)).sum().item() <= 2


def _normals_ref(Ws, bs, feat, X, Y, Z, cal, R, box):
    """surface_normals restated: the world points colorization() samples, the fp64 gradient there, -(g * L/R * (1,1,-1))
    normalised; zero where the gradient vanishes or is undefined"""
    lo, hi = torch.tensor(box[0], dtype=torch.float32), torch.tensor(box[1], dtype=torch.float32)
    verts = torch.stack([X.float(), Y.float(), R - Z.float()], 1)
    world = verts * ((hi - lo) / R)[None] + lo[None]
    _, g = query_grad_ref(feat, world.t().contiguous(), cal, Ws, bs, spec.LAST_SIGMOID, dtype=torch.float64)
    axis = (hi - lo).double() / R * torch.tensor([1.0, 1.0, -1.0], dtype=torch.float64)
    n = -(g.t() * axis)
    norm = n.norm(dim=1, keepdim=True)
    return torch.where(norm > 0, n / norm.clamp_min(1e-300), torch.zeros_like(n))


def test_surface_render_and_normals_over_a_box_with_nan_depths():
    """Visible vertices of a {0,1} ball cut by the volume's faces: a column whose first occupied node lies at k < 2 has a
    NaN depth.  The colour image (tensor-core and exact routes) is the restatement's to 1e-4 with the same NaN pixels; the
    analytic normals (fp32, tc, auto) are the fp64 restatement's within their bars, and exactly zero at NaN-depth vertices."""
    from monoport_b200.recon import colorization, forward_vertices, surface_normals
    R = 65
    vol = torch.from_numpy(spec.analytic_volume(R, "ball01"))[None, None]
    X, Y, Z, _ = forward_vertices(vol.cuda(), "front")
    nan = torch.isnan(Z).cpu()
    assert 0 < int(nan.sum()) < Z.numel()
    cal = spec.scene_calib(20, 33)
    Wc, bc = spec.make_weights(spec.C_CHANNELS, 21)
    netC = build_net("C", Wc, bc)
    featc = spec.make_feat(512, 128, 128, 22)

    def qc(points, calib):
        return spec.query_ref(featc, points, calib, Wc, bc, spec.LAST_TANH)
    want = spec.colorization_ref(qc, X.cpu(), Y.cpu(), Z.cpu(), cal, resolution=R, b_min=B1[0], b_max=B1[1])
    assert bool(torch.isnan(want).any())
    for precision in ("auto", "fp32"):
        netC.precision = precision
        img = colorization(netC, [[featc.cuda()]], X, Y, Z, cal.cuda(), resolution=R, b_min=B1[0], b_max=B1[1]).cpu()
        assert torch.equal(torch.isnan(img), torch.isnan(want)), precision
        ok = ~torch.isnan(want)
        assert (img[ok] - want[ok]).abs().max().item() <= 1e-4, precision
    Ws, bs = spec.make_weights(spec.G_CHANNELS, 1234)
    net = build_net("G", Ws, bs)
    feat = spec.make_feat(256, 128, 128, 77)
    n64 = _normals_ref(Ws, bs, feat, X.cpu(), Y.cpu(), Z.cpu(), cal, R, B1)
    fin = ~nan
    assert int((n64[fin].norm(dim=1) > 0.5).sum()) > 100
    bars = {"fp32": (1e-5, 1e-3), "tc": (1e-3, 5e-2), "auto": (1e-3, 5e-2)}
    for precision, (med_bar, p99_bar) in bars.items():
        n = surface_normals(net, [[feat.cuda()]], X, Y, Z, cal.cuda(), R, B1[0], B1[1], precision=precision).cpu()
        assert bool((n[nan] == 0).all()), precision
        err = (n[fin].double() - n64[fin]).abs().flatten()
        med, p99 = err.median().item(), torch.quantile(err, 0.99).item()
        print("normals %s over the box: |err| median %.2e, p99 %.2e, max %.2e" % (precision, med, p99, err.max().item()))
        assert med <= med_bar and p99 <= p99_bar, (precision, med, p99)


@pytest.mark.parametrize("faster", [True, False])
def test_frame_graph_ring_over_a_box_equals_the_eager_chain(faster):
    """Two captured lanes over the box with netC, the analytic normal image and the mesh with its normals and colours: every
    frame -- the person cut by the box, an empty frame, another person -- equals the eager chain with the same box bit for
    bit (NaNs compared as NaN): engine -> forward_vertices -> colorization / surface_normals("auto"), and
    reconstruction(engine=...) -> mesh_normals("auto") -> mesh_colours."""
    from monoport_b200.engine import Seg3dLossless, make_query_func
    from monoport_b200.pipeline import FrameGraph, FrameGraphRing
    from monoport_b200.recon import colorization, forward_vertices, mesh_colours, mesh_normals, reconstruction, surface_normals
    net, feats, empty, _, _ = _person()
    netC = build_net("C", *spec.make_weights(spec.C_CHANNELS, 21))
    cal = spec.scene_calib(20, 33)
    eng = Seg3dLossless(make_query_func(net), *_box(), RES, balance_value=0.5, faster=faster).to("cuda")
    c0 = spec.make_feat(512, 128, 128, 22, 0.5).cuda()
    c1 = spec.make_feat(512, 128, 128, 23, 0.5).cuda()
    fat = feats[1].clone()
    fat[0, 0] += 0.6                                     # a thicker, wider person: the box cuts it
    frames = [(feats[0], c0), (fat, c0), (empty, c1), (feats[1], c1)]
    R = RES[-1]
    want = []
    for f, c in frames:
        sdf = eng(im_feat_list=[[f]], calib_tensor=cal.cuda())
        if sdf is None:
            want.append(None)
            continue
        sdf = sdf.clone()
        X, Y, Z, N = forward_vertices(sdf, "front")
        Ng = surface_normals(net, [[f]], X, Y, Z, cal.cuda(), R, B1[0], B1[1], precision="auto")
        rnorm = colorization(netC, None, X, Y, Z, cal.cuda(), norm=Ng, resolution=R)
        rtex = colorization(netC, [[c]], X, Y, Z, cal.cuda(), resolution=R, b_min=B1[0], b_max=B1[1])
        verts, faces, _, _ = reconstruction(net, "cuda", cal.cuda(), R, B1[0], B1[1], use_octree=True, feats=[[f]], engine=eng)
        want.append((sdf, X, Y, Z, N, rnorm, rtex, verts, faces, mesh_normals(net, [[f]], verts, cal.cuda(), "auto"),
                     mesh_colours(netC, [[c]], verts, cal.cuda())))
    assert want[2] is None and all(w is not None for k, w in enumerate(want) if k != 2)
    occ = want[1][0][0, 0] > 0.5                         # the cut frame reaches the volume's faces
    assert bool(occ[0].any() and occ[-1].any() and occ[:, 0].any() and occ[:, :, 0].any())
    ring = FrameGraphRing(lambda: FrameGraph(net, eng, cal, "front", with_encoder=False, netC=netC, render_normals="gradient",
                                             mesh=True, mesh_normals=True, mesh_colours=True), n_lanes=2)
    n_out = 0
    for i, (w, out) in enumerate(zip(want, ring.run(iter(frames)))):
        n_out += 1
        assert len(out) == 11
        if w is None:
            assert all(t is None for t in out)
            continue
        for k, (a, b) in enumerate(zip(w, out)):
            assert _same(a, b), (i, k)
    assert n_out == len(frames)
    ring.close()


def test_frame_graph_ring_with_the_topk_engine():
    """A Seg3dTopk lane pair: every frame, the empty one included, returns what the eager top-k engine and forward_vertices
    return, and the same per-level counts."""
    from monoport_b200.engine import Seg3dTopk, make_query_func
    from monoport_b200.pipeline import FrameGraph, FrameGraphRing
    from monoport_b200.recon import forward_vertices
    net, feats, empty, _, _ = _person()
    cal = spec.scene_calib(20, 33)
    eng = Seg3dTopk(make_query_func(net), *_box(), RES, [0, 9000, 30000]).to("cuda")
    frames = [feats[0], empty, feats[1], empty]
    want = []
    for f in frames:
        sdf = eng(im_feat_list=[[f]], calib_tensor=cal.cuda())
        sdf = None if sdf is None else sdf.clone()
        want.append(((sdf,) + tuple(forward_vertices(sdf, "front")), list(eng.last_stats)))
    assert want[1][1] == [17 ** 3, 0, 0] and want[0][1] == [17 ** 3, 9000, 30000]
    ring = FrameGraphRing(lambda: FrameGraph(net, eng, cal, "front", with_encoder=False), n_lanes=2)
    for i, ((w, stats), out) in enumerate(zip(want, ring.run(iter(frames)))):
        for k, (a, b) in enumerate(zip(w, out)):
            assert _same(a, b), (i, k)
        assert ring.lanes[i % 2].last_stats == stats, (i, ring.lanes[i % 2].last_stats, stats)
    ring.close()
