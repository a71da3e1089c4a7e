"""GPU tier of the head goldens (tests/golden/head_*.npz): heads other than the two shipped ones through every entry point
of the library -- query(), the grid queries, a batch, the host-buffer query, the point gradient, colorization(),
surface_normals(), the octree engines and the captured frame -- against the reference and, bit for bit, against each other:
"auto" must be the exact kernel for every head the tensor-core programs do not run.  The tile sizes follow the device's
shared-memory opt-in.  no_residual heads are refused everywhere.  On the shipped widths, the tensor-core programs' default
feature limit per last op."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import spec
from grad_cases import within_bar
from head_cases import (build_head_net, fp32_tile, head_cases, head_grad_cases, head_widths, load_head_case,
                        load_head_grad_case, shipped_widths)

pytestmark = pytest.mark.gpu

B_MIN, B_MAX = (-1.0, -1.0, -1.0), (1.0, 1.0, 1.0)
FP32_HEADS = [n for n in head_cases() if shipped_widths(head_widths(n)) is None]
TC_PAIR_HEADS = [n for n in head_cases() if shipped_widths(head_widths(n)) is not None]
DEFAULT_LIMIT = {("G", spec.LAST_NONE): 3.0, ("G", spec.LAST_TANH): 3.0, ("C", spec.LAST_SIGMOID): 12.0,
                 ("C", spec.LAST_NONE): 4.0}


def _cuda(c):
    return c["feat"].cuda(), c["points"].cuda(), (c["calib"].cuda() if c["calib"] is not None else None)


def _bar(got, want):
    return (got.cpu() - want).abs().max().item() <= 2e-5 * max(1.0, want.abs().max().item())


def _query(net, feat, pts, cal, mode):
    net.precision = mode
    return net.query([[feat]], pts, calibs=cal)[0].clone()


def _optin():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).shared_memory_per_block_optin


# ---- query() and the routes that must equal it ---------------------------------------------------------------------------
@pytest.mark.parametrize("name", FP32_HEADS)
def test_query_matches_head_golden_and_auto_is_the_exact_kernel(name):
    c = load_head_case(name)
    if fp32_tile(c["chans"], _optin()) is None:
        pytest.skip("this device's shared-memory opt-in does not fit the head")
    net = build_head_net(c)
    assert not net.surface_classifier.tc_supported()
    feat, pts, cal = _cuda(c)
    exact = _query(net, feat, pts, cal, "fp32")
    assert _bar(exact[0], c["expected"]), (exact[0].cpu() - c["expected"]).abs().max().item()
    zero = c["expected"] == 0
    assert bool(zero.any()) and torch.equal(exact[0].cpu()[zero], c["expected"][zero]), "out-of-image points must be 0"
    assert torch.equal(_query(net, feat, pts, cal, "auto"), exact)
    net.precision = "tc"
    with pytest.raises(RuntimeError):
        net.query([[feat]], pts, calibs=cal)


@pytest.mark.parametrize("name", [n for n in FP32_HEADS if n != "p8_full"])
def test_grid_batch_and_host_queries_equal_the_point_query(name):
    """query_grid (single-output heads) == query() of the grid's points; a B = 3 batch == the three single queries; the
    host-buffer entry point == query(); in "fp32" and "auto", bit for bit."""
    from monoport_b200 import _lib
    c = load_head_case(name)
    net = build_head_net(c)
    feat, pts, cal = _cuda(c)
    res = c["chans"][-1]
    feats = torch.cat([feat, -0.5 * feat, feat.flip(3)], 0)
    bpts = torch.cat([pts, pts.flip(2), pts * 0.9], 0)
    bcal = cal.expand(3, 4, 4).contiguous() if cal is not None else None
    R = 9
    world = spec.level_points(spec._grid_coords(R, 1), R, B_MIN, B_MAX).t().contiguous()[None].cuda()
    for mode in ("fp32", "auto"):
        one = _query(net, feat, pts, cal, mode)
        if res == 1:
            vol = net.query_grid(feat, cal, R, B_MIN, B_MAX)
            assert torch.equal(vol.reshape(-1), _query(net, feat, world, cal, mode)[0, 0]), mode
        got = net.query([[feats]], bpts, calibs=bcal)[0]
        for b in range(3):
            want = _query(net, feats[b:b + 1], bpts[b:b + 1], bcal[b:b + 1] if bcal is not None else None, mode)
            assert torch.equal(got[b:b + 1], want), (mode, b)
        lib = _lib.load()
        fh = ctypes.c_void_p()
        _lib.check(lib.mp_feat_create(feat.shape[1], c["H"], c["W"], ctypes.byref(fh)))
        p = c["points"][0].contiguous().numpy()
        n = p.shape[1]
        out = np.empty((res, n), dtype=np.float32)
        f = c["feat"].contiguous().numpy()
        proj = _lib.PROJ_PERSPECTIVE if c["proj"] == "perspective" else _lib.PROJ_ORTHOGONAL
        _lib.check(lib.mp_query_points_host(net.surface_classifier.handle(), fh, f.ctypes.data_as(ctypes.c_void_p),
                                            p.ctypes.data_as(ctypes.c_void_p), n, _lib.calib12(c["calib"]), proj,
                                            ctypes.c_float(spec.Z_SCALE), out.ctypes.data_as(ctypes.c_void_p),
                                            _lib.MODE_AUTO if mode == "auto" else _lib.MODE_FP32, None))
        lib.mp_feat_destroy(fh)
        assert torch.equal(torch.from_numpy(out), one[0].cpu()), mode


@pytest.mark.parametrize("name", head_grad_cases())
def test_gradient_matches_head_golden(name):
    """query_gradient: its value query()'s bit for bit, the gradient within its bar of the reference's fp32 autograd;
    "auto" the exact program bit for bit; "tc" refused"""
    c = load_head_grad_case(name)
    net = build_head_net(c)
    feat, pts, cal = _cuda(c)
    val, dp = net.query_gradient([[feat]], pts, calibs=cal)
    assert torch.equal(val, _query(net, feat, pts, cal, "fp32"))
    assert _bar(val[0], c["value"])
    ok, msg = within_bar(dp[0].cpu(), c["grad32"])
    assert ok, msg
    va, da = net.query_gradient([[feat]], pts, calibs=cal, precision="auto")
    assert torch.equal(va, val) and torch.equal(da, dp)
    with pytest.raises(RuntimeError):
        net.query_gradient([[feat]], pts, calibs=cal, precision="tc")


def _vertices(R=33):
    from monoport_b200.recon import forward_vertices
    vol = torch.from_numpy(spec.analytic_volume(R, "sphere"))[None, None].cuda()
    X, Y, Z, _ = forward_vertices(vol, "front")
    return X, Y, Z


@pytest.mark.parametrize("name", ["single", "g_res3"])
def test_colorization_with_a_three_output_head(name):
    """colorization() through a non-shipped 3-output head: the restatement within 2e-5, "auto" == "fp32" bit for bit"""
    from monoport_b200.recon import colorization
    c = load_head_case(name)
    netC = build_head_net(c)
    calib = c["calib"] if c["calib"] is not None else torch.eye(4)[None]     # colorization() takes a camera
    feat, cal = c["feat"].cuda(), calib.cuda()
    X, Y, Z = _vertices()
    netC.precision = "fp32"
    exact = colorization(netC, [[feat]], X, Y, Z, cal, resolution=33)

    def qc(points, calib):
        return spec.query_ref(c["feat"], points, calib, c["Ws"], c["bs"], c["last_op"], c["proj"])

    want = spec.colorization_ref(qc, X.cpu(), Y.cpu(), Z.cpu(), calib, resolution=33)
    assert (exact.cpu() - want).abs().max().item() <= 2e-5
    netC.precision = "auto"
    assert torch.equal(colorization(netC, [[feat]], X, Y, Z, cal, resolution=33), exact)


@pytest.mark.parametrize("name", ["narrow", "deep", "g128"])
def test_surface_normals_auto_is_the_exact_gradient(name):
    """surface_normals(precision="auto") -- the device route, mp_surface_normals_async -- is that route in the exact mode
    bit for bit, and the normalised exact gradient of precision="fp32" (which normalises in torch) up to rounding"""
    from monoport_b200.recon import _surface_normals_device, surface_normals
    c = load_head_case(name)
    net = build_head_net(c)
    feat, _, cal = _cuda(c)
    X, Y, Z = _vertices()
    auto = surface_normals(net, [[feat]], X, Y, Z, cal, resolution=33, precision="auto")
    assert torch.equal(auto, _surface_normals_device(net, feat, X, Y, Z, cal, 33, B_MIN, B_MAX, "fp32"))
    exact = surface_normals(net, [[feat]], X, Y, Z, cal, resolution=33, precision="fp32")
    assert (auto - exact).abs().max().item() <= 1e-6 and bool((exact.norm(dim=1) > 0.5).any())


# ---- tile fits ----------------------------------------------------------------------------------------------------------
def _zero_head(chans):
    return dict(chans=chans, last_op=spec.LAST_SIGMOID, Ws=[torch.zeros(chans[l + 1], chans[l] + (chans[0] if l else 0))
                                                             for l in range(len(chans) - 1)],
                bs=[torch.zeros(chans[l + 1]) for l in range(len(chans) - 1)], proj="orthogonal")


def test_tile_fits_follow_the_device_opt_in():
    """The exactly full P = 32 and P = 8 heads run (their parity: the golden tests), the next width up takes the next
    tile or is refused, and the gradient of the P = 8 head is refused -- as the footprint predicts for this device's
    shared-memory opt-in, read from the device."""
    optin = _optin()
    cases = [([1025, 512, 255, 1], False), ([1025, 512, 256, 1], False), ([1025, 4096, 2071, 1], False),
             ([1025, 4096, 2072, 1], False), ([1025, 4096, 2071, 1], True), ([1025, 512, 255, 1], True),
             # the gradient's tiles 32, 16 and 8 exactly full, and one more unit in the second hidden layer
             ([129, 1024, 587, 1], True), ([129, 1024, 588, 1], True), ([513, 2048, 936, 1], True),
             ([513, 2048, 937, 1], True), ([1025, 4096, 1883, 1], True), ([1025, 4096, 1884, 1], True)]
    if optin == 232448:
        assert [fp32_tile(ch, optin, g) for ch, g in cases] == [32, 16, 8, None, None, 16, 32, 16, 16, 8, 8, None]
    pts = torch.zeros(1, 3, 40, device="cuda")
    for chans, grad in cases:
        feat = torch.zeros(1, chans[0] - 1, 5, 4, device="cuda")
        net = build_head_net(_zero_head(chans))
        call = (lambda: net.query_gradient([[feat]], pts)) if grad else (lambda: net.query([[feat]], pts))
        net.precision = "fp32"
        if fp32_tile(chans, optin, grad) is None:
            with pytest.raises(RuntimeError, match="head too wide for the (fp32|gradient) kernel"):
                call()
        else:
            out = call()
            torch.cuda.synchronize()
            assert bool((out[0] == 0.5).all()), chans              # zero weights: sigmoid(0) at every point (all in the image)


# ---- the engines and the captured frame ----------------------------------------------------------------------------------
def _person(c_like, seed=3):
    """a height-field person through the widths of the g128 golden (spec.heightfield_person's wiring)"""
    chans = head_widths(c_like)
    Ws, bs = spec.make_weights(chans, seed)
    Ws, bs, feat, _ = spec.heightfield_person(Ws, bs, spec.make_feat(chans[0] - 1, 64, 80, seed + 1, 0.5))
    c = dict(chans=chans, last_op=spec.LAST_SIGMOID, Ws=Ws, bs=bs, proj="orthogonal")
    return build_head_net(c), feat.cuda()


def _nets():
    """(net, feature map) pairs: the g128 person and the narrow golden head"""
    person = _person("g128")
    c = load_head_case("narrow")
    return [person, (build_head_net(c), c["feat"].cuda())]


@pytest.mark.parametrize("kind", ["faster", "lossless", "topk"])
def test_fused_engines_equal_the_callback_engines(kind):
    from monoport_b200.engine import Seg3dLossless, Seg3dTopk, make_query_func
    b = np.array([[-1.0, -1.0, -1.0]], dtype=np.float32)
    res = [9, 17, 33]
    cal = spec.scene_calib(20, 33).cuda()
    for net, feat in _nets():
        assert not net.surface_classifier.tc_supported()

        def plain(points, im_feat_list, calib_tensor):
            return net.query(im_feat_list, points=points.permute(0, 2, 1), calibs=calib_tensor)[0]

        def make(fn):
            if kind == "topk":
                return Seg3dTopk(fn, b, -b, res, num_points=[100, 200, 400], balance_value=0.5).to("cuda")
            return Seg3dLossless(fn, b, -b, res, balance_value=0.5, faster=kind == "faster").to("cuda")

        for mode in ("fp32", "auto"):
            net.precision = mode
            fused, generic = make(make_query_func(net)), make(plain)
            a = fused(im_feat_list=[[feat]], calib_tensor=cal)
            g = generic(im_feat_list=[[feat]], calib_tensor=cal)
            assert (a is None) == (g is None) and fused.last_stats == generic.last_stats, (kind, mode)
            assert a is None or torch.equal(a, g), (kind, mode)


def test_frame_graph_with_non_shipped_heads_equals_the_eager_chain():
    """A FrameGraph ring with the g128 person as netG and the one-layer 3-output head as netC (analytic normal image,
    colour image, mesh normals and mesh colours): every frame equals the eager chain bit for bit."""
    from monoport_b200.engine import Seg3dLossless, make_query_func
    from monoport_b200.pipeline import FrameGraph, FrameGraphRing
    from monoport_b200.recon import colorization, forward_vertices, mesh_colours, mesh_normals, reconstruction, surface_normals
    net, feat = _person("g128")
    c = load_head_case("single")
    netC = build_head_net(c)
    b = np.array([[-1.0, -1.0, -1.0]], dtype=np.float32)
    eng = Seg3dLossless(make_query_func(net), b, -b, [17, 33, 65], balance_value=0.5, faster=True).to("cuda")
    cal = spec.scene_calib(20, 33)
    c0 = spec.make_feat(c["chans"][0] - 1, feat.shape[2], feat.shape[3], 31).cuda()    # netC's map: netG's H x W
    c1 = torch.flip(c0, (3,)) * 0.5
    empty = feat.clone()
    empty[0, 0] = -5.0
    frames = [(feat, c0), (empty, c0), (feat * 1.05, c1)]
    want = []
    for f, cf in frames:
        sdf = eng(im_feat_list=[[f]], calib_tensor=cal.cuda())
        X, Y, Z, _ = forward_vertices(sdf, "front")
        if X is None:
            want.append(None)
            continue
        N = surface_normals(net, [[f]], X, Y, Z, cal.cuda(), resolution=65, precision="auto")
        rnorm = colorization(netC, None, X, Y, Z, cal.cuda(), norm=N, resolution=65)
        rtex = colorization(netC, [[cf]], X, Y, Z, cal.cuda(), resolution=65)
        verts, faces, _, _ = reconstruction(net, "cuda", cal.cuda(), 65, B_MIN, B_MAX, use_octree=True, feats=[[f]], engine=eng)
        want.append((sdf.clone(), X, Y, Z, rnorm, rtex, verts, faces,
                     mesh_normals(net, [[f]], verts, cal.cuda(), precision="auto"), mesh_colours(netC, [[cf]], verts, cal.cuda())))
    assert want[1] is None and want[0] is not None and want[2] is not None
    ring = FrameGraphRing(lambda: FrameGraph(net, eng, cal, "front", with_encoder=False, input_shape=tuple(feat.shape),
                                             netC=netC, render_normals="gradient", mesh=True, mesh_normals=True,
                                             mesh_colours=True), n_lanes=2)
    n_out = 0
    for i, (w, out) in enumerate(zip(want, ring.run(iter(frames)))):
        n_out += 1
        assert len(out) == 11
        if w is None:
            assert all(t is None for t in out)
            continue
        got = out[:4] + out[5:]
        for k, (a, g) in enumerate(zip(w, got)):
            assert a.shape == g.shape and torch.equal(a, g), (i, k)
    assert n_out == len(frames)
    ring.close()


# ---- no_residual heads are refused ---------------------------------------------------------------------------------------
def test_no_residual_head_is_refused_everywhere_and_writes_nothing():
    from monoport_b200.engine import Seg3dLossless, make_query_func
    from monoport_b200.pipeline import FrameGraph
    from monoport_b200.recon import colorization
    c = load_head_case("narrow")
    net = build_head_net(c, no_residual=True)
    cs = load_head_case("single")
    netC = build_head_net(dict(cs, chans=[65, 64, 3]), no_residual=True)
    feat, pts, cal = _cuda(c)
    msg = "no_residual heads are not supported"
    with pytest.raises(RuntimeError, match=msg):
        net.query([[feat]], pts, calibs=cal)
    with pytest.raises(RuntimeError, match=msg):
        net.query_gradient([[feat]], pts, calibs=cal)
    vol = torch.full((9, 9, 9), -7.0, device="cuda")
    with pytest.raises(RuntimeError, match=msg):
        net.query_grid(feat, cal, 9, B_MIN, B_MAX, out=vol)
    assert bool((vol == -7.0).all()), "a refused grid query must write nothing"
    X, Y, Z = _vertices()
    with pytest.raises(RuntimeError, match=msg):
        colorization(netC, [[cs["feat"].cuda()]], X, Y, Z, torch.eye(4, device="cuda")[None], resolution=33)
    b = np.array([[-1.0, -1.0, -1.0]], dtype=np.float32)
    eng = Seg3dLossless(make_query_func(net), b, -b, [9, 17], balance_value=0.5, faster=True).to("cuda")
    with pytest.raises(RuntimeError, match=msg):
        eng(im_feat_list=[[feat]], calib_tensor=cal)
    with pytest.raises(RuntimeError, match=msg):
        FrameGraph(net, eng, spec.scene_calib(20, 33), "front", with_encoder=False)


# ---- the feature limit per last op on the shipped widths -----------------------------------------------------------------
def _below(a):
    return float(np.nextafter(np.float32(a), np.float32(0)))


@pytest.mark.parametrize("name", TC_PAIR_HEADS)
def test_feature_limit_of_each_last_op(name):
    """A map at 0.99 x the head's default limit: "auto" runs the tensor cores (not the fp32 bits) within 1e-4 of the
    reference.  The same map just above the default limit, or the limit set just below its max |feature|: "auto" is the
    exact kernel, bit for bit."""
    c = load_head_case(name)
    limit = DEFAULT_LIMIT[(c["net"], c["last_op"])]
    assert c["amax"] == pytest.approx(0.99 * limit)
    net = build_head_net(c)
    if not net.surface_classifier.tc_supported():
        pytest.skip("no tensor-core program on this device")
    feat, pts, cal = _cuda(c)
    exact = _query(net, feat, pts, cal, "fp32")
    assert _bar(exact[0], c["expected"])
    auto = _query(net, feat, pts, cal, "auto")
    assert not torch.equal(auto, exact)
    assert (auto[0].cpu() - c["expected"]).abs().max().item() <= 1e-4
    above = feat * (1.001 / 0.99)
    assert above.abs().max().item() > limit
    assert torch.equal(_query(net, above, pts, cal, "auto"), _query(net, above, pts, cal, "fp32"))
    net.surface_classifier.tc_feature_limit = _below(feat.abs().max().item())
    assert torch.equal(_query(net, feat, pts, cal, "auto"), exact)
