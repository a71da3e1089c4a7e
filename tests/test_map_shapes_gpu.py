"""GPU tier of the map-shape goldens (tests/golden/shape_*.npz): query(), the grid queries, the batched query, the point
gradient, the octree engine and the colour renders on feature maps that are not square, whose texel count is not a multiple
of 128, that have an axis of length 1, or that sit at or above the tensor-core program's 65536 texels -- against the
reference, and against the other routes of the library bit for bit.  Also both sides of the range guard's limit."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import spec
from grad_cases import within_bar
from helpers import build_net
from shape_cases import (TC_TEXEL_LIMIT, load_shape_batch_case, load_shape_case, load_shape_grad_case, shape_cases,
                         shape_grad_cases, within_fp32_bar)

pytestmark = pytest.mark.gpu

TOL = {"fp32": 2e-5, "tc": 1e-4, "auto": 1e-4}
B_MIN, B_MAX = (-1.0, -1.0, -1.0), (1.0, 1.0, 1.0)


def _modes(net, c):
    """every precision that runs this map: "tc" only up to the tensor-core program's texel limit"""
    tc = net.surface_classifier.tc_supported() and c["H"] * c["W"] <= TC_TEXEL_LIMIT
    return ["fp32", "tc", "auto"] if tc else ["fp32", "auto"]


def _cuda(c):
    return c["feat"].cuda(), c["points"].cuda(), (c["calib"].cuda() if c["calib"] is not None else None)


@pytest.mark.parametrize("name", shape_cases())
def test_query_matches_reference_shape_golden(name):
    c = load_shape_case(name)
    net = build_net(c)
    feat, pts, cal = _cuda(c)
    for mode in _modes(net, c):
        net.precision = mode
        got = net.query([[torch.zeros_like(feat)]] * 3 + [[feat]], pts, calibs=cal)[0][0].cpu()
        err = (got - c["expected"]).abs().max().item()
        if mode == "fp32":
            ok, msg = within_fp32_bar(got, c)
            assert ok, (name, msg)
        else:
            assert err <= TOL[mode], (name, mode, err)
        zero = c["expected"] == 0
        assert torch.equal(got[zero], c["expected"][zero]), "out-of-image points must be exactly 0"


@pytest.mark.parametrize("name", ["g_over", "c_over"])
def test_above_the_texel_limit_auto_is_the_exact_kernel_and_tc_refuses(name):
    """A map of more than 65536 texels: "auto" returns what "fp32" returns, bit for bit, for points and (geometry head) for
    the dense grid and a node range of it; "tc" refuses with an error that names the limit."""
    c = load_shape_case(name)
    assert c["H"] * c["W"] > TC_TEXEL_LIMIT
    net = build_net(c)
    if not net.surface_classifier.tc_supported():
        pytest.skip("no tensor-core program on this device")
    feat, pts, cal = _cuda(c)
    R = 33
    calls = {"points": lambda: net.query([[feat]], pts, calibs=cal)[0]}
    if c["net"] == "G":
        calls["grid"] = lambda: net.query_grid(feat, cal, R, B_MIN, B_MAX)
        calls["grid_range"] = lambda: net.query_grid_range(feat, cal, R, B_MIN, B_MAX, 1000, 20000)
    for what, call in calls.items():
        net.precision = "fp32"
        exact = call().clone()
        net.precision = "auto"
        assert torch.equal(call(), exact), what
        net.precision = "tc"
        with pytest.raises(RuntimeError, match="at most 65536 texels"):
            call()


def test_grid_equals_points_and_slabs_tile_on_a_non_square_map():
    c = load_shape_case("g_wide")
    net = build_net(c)
    feat, _, cal = _cuda(c)
    R = 21
    world = spec.level_points(spec._grid_coords(R, 1), R, B_MIN, B_MAX)          # [N,3]
    want = spec.query_ref(c["feat"], world.t().contiguous(), c["calib"], c["Ws"], c["bs"], spec.LAST_SIGMOID)[0]
    for mode in _modes(net, c):
        net.precision = mode
        vol = net.query_grid(feat, cal, R, B_MIN, B_MAX)
        assert (vol.reshape(-1).cpu() - want).abs().max().item() <= TOL[mode], mode
        pts = net.query([[feat]], world.t().contiguous()[None].cuda(), calibs=cal)[0][0, 0]
        assert torch.equal(pts, vol.reshape(-1)), mode
        slabs = [net.query_grid(feat, cal, R, B_MIN, B_MAX, z0=z0, nz=nz) for z0, nz in ((0, 4), (4, 9), (13, 8))]
        assert torch.equal(torch.cat(slabs, 0), vol), mode
        ranges = [net.query_grid_range(feat, cal, R, B_MIN, B_MAX, a, b - a) for a, b in ((0, 1000), (1000, 5003), (5003, R ** 3))]
        assert torch.equal(torch.cat(ranges), vol.reshape(-1)), mode


def test_channels_last_non_square_map_equals_contiguous_upload():
    """A channels_last map (bound in place, read as [H][W][C]) against the contiguous upload, single and batched."""
    c = load_shape_case("g_wide")
    net = build_net(c)
    feat, pts, cal = _cuda(c)
    feat_cl = feat.contiguous(memory_format=torch.channels_last)
    assert not feat_cl.is_contiguous() and torch.equal(feat_cl, feat)
    cb = load_shape_batch_case("g_wide_persp")
    netb = build_net(cb)
    fb, pb, calb = _cuda(cb)
    fb_cl = fb.contiguous(memory_format=torch.channels_last)
    assert not fb_cl.is_contiguous()
    for mode in _modes(net, c):
        net.precision = mode
        a = net.query([[feat]], pts, calibs=cal)[0].clone()
        assert torch.equal(net.query([[feat_cl]], pts, calibs=cal)[0], a), mode
        netb.precision = mode
        a = netb.query([[fb]], pb, calibs=calb)[0].clone()
        assert torch.equal(netb.query([[fb_cl]], pb, calibs=calb)[0], a), mode


def test_batched_non_square_maps_equal_single_queries():
    """Three 72 x 136 maps (each ends in a partial 128-texel block) with their own perspective cameras: within the bar of the
    batched golden, and image b equal to the single query of image b, bit for bit, in every mode."""
    c = load_shape_batch_case("g_wide_persp")
    net = build_net(c)
    feat, pts, cal = _cuda(c)
    for mode in _modes(net, c):
        net.precision = mode
        got = net.query([[feat]], pts, calibs=cal)[0].clone()
        assert (got.cpu() - c["expected"]).abs().max().item() <= TOL[mode], mode
        zero = c["expected"] == 0
        assert torch.equal(got.cpu()[zero], c["expected"][zero])
        for b in range(c["B"]):
            one = net.query([[feat[b:b + 1]]], pts[b:b + 1], calibs=cal[b:b + 1])[0][0]
            assert torch.equal(got[b], one), (mode, b)


@pytest.mark.parametrize("name", shape_grad_cases())
def test_gradient_matches_reference_shape_golden(name):
    c = load_shape_grad_case(name)
    net = build_net(c)
    feat, pts, cal = _cuda(c)
    val, dp = net.query_gradient([[feat]], pts, calibs=cal)
    net.precision = "fp32"
    assert torch.equal(val, net.query([[feat]], pts, calibs=cal)[0])
    assert (val[0].cpu() - c["value"]).abs().max().item() <= 2e-5
    ok, msg = within_bar(dp[0].cpu(), c["grad32"])
    assert ok, msg


def test_fused_engine_equals_generic_engine_on_a_non_square_map():
    """The occupancy engine on a 96 x 160 height-field person: the fused on-device pyramid equals the Python-callback pyramid
    driven by query(), bit for bit (the same kernel evaluates the same points)."""
    from monoport_b200.engine import Seg3dLossless, make_query_func
    Ws, bs = spec.make_weights(spec.G_CHANNELS, 3)
    Ws, bs, feat, _ = spec.heightfield_person(Ws, bs, spec.make_feat(256, 96, 160, 4, 0.5))
    net = build_net("G", Ws, bs)
    cal = spec.scene_calib(20, 33).cuda()
    feats = [[feat.cuda()]]
    b = np.array([[-1.0, -1.0, -1.0]], dtype=np.float32)
    res = [17, 33, 65]
    for mode in (["fp32", "tc"] if net.surface_classifier.tc_supported() else ["fp32"]):
        net.precision = mode
        fused = Seg3dLossless(make_query_func(net), b, -b, res, balance_value=0.5, faster=True).to("cuda")

        def plain(points, im_feat_list, calib_tensor):
            return net.query(im_feat_list, points=points.permute(0, 2, 1), calibs=calib_tensor)[0]

        generic = Seg3dLossless(plain, b, -b, res, balance_value=0.5, faster=True).to("cuda")
        a = fused(im_feat_list=feats, calib_tensor=cal)
        g = generic(im_feat_list=feats, calib_tensor=cal)
        assert a is not None and g is not None and bool((a > 0.5).any())
        assert fused.last_stats == generic.last_stats, mode
        assert torch.equal(a, g), mode


# ---- the colour renders --------------------------------------------------------------------------------------------------
def _vertices(R=65):
    from monoport_b200.recon import forward_vertices
    vol = torch.from_numpy(spec.analytic_volume(R, "ellipsoid"))[None, None].cuda()
    X, Y, Z, _ = forward_vertices(vol, "front")
    return X, Y, Z


def _render_async(netC, featc, X, Y, Z, cal, R, mode):
    """mp_colorize_surface_async, the vertex count on the device"""
    from monoport_b200 import _lib
    count = torch.tensor([X.numel()], dtype=torch.int64, device="cuda")
    img = torch.ones((R, R, 3), dtype=torch.float32, device="cuda")
    fh = netC.feature_handle(featc)
    _lib.check(_lib.load().mp_colorize_surface_async(
        netC.surface_classifier.handle(), fh.ptr, ctypes.c_void_p(X.contiguous().data_ptr()),
        ctypes.c_void_p(Y.contiguous().data_ptr()), ctypes.c_void_p(Z.float().contiguous().data_ptr()),
        ctypes.c_void_p(count.data_ptr()), X.numel(), R, _lib.f3(B_MIN), _lib.f3(B_MAX), _lib.calib12(cal), _lib.PROJ_ORTHOGONAL,
        ctypes.c_float(netC.normalizer.scale), mode, ctypes.c_void_p(img.data_ptr()), _lib.stream_ptr()),
        "mp_colorize_surface_async")
    torch.cuda.synchronize()
    return img


def _colour_want(c, X, Y, Z, R=65):
    def qc(points, calib):
        return spec.query_ref(c["feat"], points, calib, c["Ws"], c["bs"], spec.LAST_TANH)
    return spec.colorization_ref(qc, X.cpu(), Y.cpu(), Z.cpu(), c["calib"], resolution=R)


def test_colorization_on_a_non_square_map():
    """Eager colorization() through the colour head on the 88 x 120 map (tensor-core program) against the restatement, and
    the enqueue-only render of the same frame bit for bit."""
    from monoport_b200 import _lib
    from monoport_b200.recon import colorization
    c = load_shape_case("c_wide")
    netC = build_net(c)
    feat, _, cal = _cuda(c)
    X, Y, Z = _vertices()
    eager = colorization(netC, [[feat]], X, Y, Z, cal, resolution=65)
    assert (eager.cpu() - _colour_want(c, X, Y, Z)).abs().max().item() <= 5e-5
    assert torch.equal(_render_async(netC, feat, X, Y, Z, cal, 65, _lib.MODE_AUTO), eager)


def test_colorization_above_the_texel_limit():
    """A 260 x 256 colour map, above the tensor-core program's texels: eager colorization() in "auto" takes the exact route
    -- within the fp32 bar of the restatement and bit for bit the enqueue-only render, which takes its exact twin there --, and
    with precision "tc" refuses exactly as query() does."""
    from monoport_b200 import _lib
    from monoport_b200.recon import colorization
    c = load_shape_case("c_over")
    netC = build_net(c)
    assert netC.surface_classifier.tc_supported() and c["H"] * c["W"] > TC_TEXEL_LIMIT
    feat, pts, cal = _cuda(c)
    X, Y, Z = _vertices()
    netC.precision = "auto"
    eager = colorization(netC, [[feat]], X, Y, Z, cal, resolution=65)
    assert (eager.cpu() - _colour_want(c, X, Y, Z)).abs().max().item() <= 2e-5
    assert torch.equal(_render_async(netC, feat, X, Y, Z, cal, 65, _lib.MODE_AUTO), eager)
    netC.precision = "tc"
    with pytest.raises(RuntimeError, match="at most 65536 texels") as by_query:
        netC.query([[feat]], pts, calibs=cal)
    with pytest.raises(RuntimeError) as by_colorization:
        colorization(netC, [[feat]], X, Y, Z, cal, resolution=65)
    assert str(by_colorization.value) == str(by_query.value)


# ---- the range guard at its limit ----------------------------------------------------------------------------------------
def _below(a):
    """the largest float32 below the float32 a"""
    return float(np.nextafter(np.float32(a), np.float32(0)))


def test_range_guard_boundary_single_and_batched():
    """limit == the frame's max |feature|: the frame is in range (tensor cores: not the fp32 bits, within 1e-4 of them); the
    float32 just below it: out of range (the fp32 bits).  Per image in a batch: an image at the limit takes the tensor cores,
    one above it the exact kernel."""
    c = load_shape_case("g_wide")
    net = build_net(c)
    if not net.surface_classifier.tc_supported():
        pytest.skip("no tensor-core program on this device")
    feat, pts, cal = _cuda(c)
    amax = feat.abs().max().item()
    net.precision = "fp32"
    exact = net.query([[feat]], pts, calibs=cal)[0].clone()
    net.precision = "auto"
    net.surface_classifier.tc_feature_limit = amax
    at = net.query([[feat]], pts, calibs=cal)[0].clone()
    assert not torch.equal(at, exact) and (at - exact).abs().max().item() <= 1e-4
    net.surface_classifier.tc_feature_limit = _below(amax)
    assert torch.equal(net.query([[feat]], pts, calibs=cal)[0], exact)

    cb = load_shape_batch_case("g_wide_persp")
    netb = build_net(cb)
    fb, pb, calb = _cuda(cb)
    amaxes = [fb[b].abs().max().item() for b in range(cb["B"])]
    assert len(set(amaxes)) == cb["B"]
    mid = sorted(amaxes)[1]
    singles = {}
    for mode in ("fp32", "tc"):
        netb.precision = mode
        netb.surface_classifier.tc_feature_limit = float("inf")
        singles[mode] = [netb.query([[fb[b:b + 1]]], pb[b:b + 1], calibs=calb[b:b + 1])[0][0].clone() for b in range(cb["B"])]
    netb.precision = "auto"
    for limit in (mid, _below(mid)):
        netb.surface_classifier.tc_feature_limit = limit
        got = netb.query([[fb]], pb, calibs=calb)[0]
        for b in range(cb["B"]):
            want = singles["tc" if amaxes[b] <= limit else "fp32"][b]
            assert torch.equal(got[b], want), (limit, b, amaxes[b])
            assert not torch.equal(singles["tc"][b], singles["fp32"][b])


def test_range_guard_boundary_colour_renders():
    """The eager render tests `max|feature| > limit` on the host, the enqueue-only render on the device: at the limit both
    give the tensor-core image, just below it both give the exact one."""
    from monoport_b200 import _lib
    from monoport_b200.recon import colorization
    c = load_shape_case("c_wide")
    netC = build_net(c)
    feat, _, cal = _cuda(c)
    X, Y, Z = _vertices()
    amax = feat.abs().max().item()
    netC.precision = "fp32"
    exact = colorization(netC, [[feat]], X, Y, Z, cal, resolution=65)
    netC.precision = "tc"
    netC.surface_classifier.tc_feature_limit = float("inf")
    tc = colorization(netC, [[feat]], X, Y, Z, cal, resolution=65)
    assert not torch.equal(tc, exact) and (tc - exact).abs().max().item() <= 1e-4
    netC.precision = "auto"
    for limit, want in ((amax, tc), (_below(amax), exact)):
        netC.surface_classifier.tc_feature_limit = limit
        assert torch.equal(colorization(netC, [[feat]], X, Y, Z, cal, resolution=65), want), ("eager", limit)
        assert torch.equal(_render_async(netC, feat, X, Y, Z, cal, 65, _lib.MODE_AUTO), want), ("async", limit)
