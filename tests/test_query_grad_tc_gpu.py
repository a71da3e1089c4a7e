"""GPU tests of the tensor-core point gradient (MonoPortNet.query_gradient with precision "tc" / "auto" ->
mp_query_points_grad_mode): the reference's fp64 autograd goldens, the value against query() in "tc" bit for bit, the exact
route on both sides of the head's feature limit and above the 65536-texel limit, the call handling, and the normals of the
synthetic person against the exact ones."""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle import spec
from helpers import build_net
from grad_cases import GOLDEN_CASES, load_golden, load_grad_case, tc_bar
from shape_cases import load_shape_case, load_shape_grad_case

pytestmark = pytest.mark.gpu


def _inputs(c):
    net = build_net(c)
    if not net.surface_classifier.tc_supported():
        pytest.skip("no tensor-core program on this device")
    gout = c["grad_output"][None].cuda() if c.get("grad_output") is not None else None
    cal = c["calib"].cuda() if c["calib"] is not None else None
    return net, [[c["feat"].cuda()]], c["points"].cuda(), cal, gout


@pytest.mark.parametrize("kind,name,n", GOLDEN_CASES)
def test_tc_gradient_matches_reference_grad_golden(kind, name, n):
    c = load_golden(kind, name)
    net, feats, pts, cal, gout = _inputs(c)
    for precision in ("tc", "auto"):
        val, dp = net.query_gradient(feats, pts, calibs=cal, grad_output=gout, precision=precision)
        assert (val[0].cpu() - c["value"]).abs().max().item() <= 1e-4
        ok, msg = tc_bar(dp[0].cpu(), c["grad64"], name)
        print(name, precision, msg)
        assert ok, msg
        outside = (c["value"] == 0).all(0)
        assert bool((dp[0].cpu()[:, outside] == 0).all())


@pytest.mark.parametrize("name", ["g_rot", "g_persp", "c_rot"])
def test_tc_value_is_query_tc_bit_for_bit_and_fp32_is_the_default(name):
    c = load_grad_case(name)
    net, feats, pts, cal, gout = _inputs(c)
    net.precision = "tc"
    want = net.query(feats, pts, calibs=cal)[0]
    val, _ = net.query_gradient(feats, pts, calibs=cal, grad_output=gout, precision="tc")
    assert torch.equal(val, want)
    a = net.query_gradient(feats, pts, calibs=cal, grad_output=gout)
    b = net.query_gradient(feats, pts, calibs=cal, grad_output=gout, precision="fp32")
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_both_sides_of_the_feature_limit():
    """limit == the frame's max |feature|: the tensor cores (the value is query()'s "tc" value); the float32 just below it:
    the exact kernel, bit for bit precision "fp32"."""
    c = load_shape_grad_case("g_wide")
    net, feats, pts, cal, _ = _inputs(c)
    amax = feats[0][0].abs().max().item()
    exact = net.query_gradient(feats, pts, calibs=cal, precision="fp32")
    net.precision = "tc"
    tcq = net.query(feats, pts, calibs=cal)[0].clone()
    net.surface_classifier.tc_feature_limit = amax
    for precision in ("tc", "auto"):
        at = net.query_gradient(feats, pts, calibs=cal, precision=precision)
        assert torch.equal(at[0], tcq) and not torch.equal(at[1], exact[1])
    net.surface_classifier.tc_feature_limit = float(np.nextafter(np.float32(amax), np.float32(0)))
    for precision in ("tc", "auto"):
        below = net.query_gradient(feats, pts, calibs=cal, precision=precision)
        assert torch.equal(below[0], exact[0]) and torch.equal(below[1], exact[1]), precision


def test_map_above_65536_texels():
    c = load_shape_case("g_over")                     # 257 x 256
    net = build_net(c)
    if not net.surface_classifier.tc_supported():
        pytest.skip("no tensor-core program on this device")
    feats, pts = [[c["feat"].cuda()]], c["points"].cuda()
    cal = c["calib"].cuda() if c["calib"] is not None else None
    exact = net.query_gradient(feats, pts, calibs=cal, precision="fp32")
    auto = net.query_gradient(feats, pts, calibs=cal, precision="auto")
    assert torch.equal(auto[0], exact[0]) and torch.equal(auto[1], exact[1])
    with pytest.raises(RuntimeError, match="65536 texels"):
        net.query_gradient(feats, pts, calibs=cal, precision="tc")


def test_strided_points_empty_input_and_refusals():
    from monoport_b200 import _lib
    c = load_grad_case("c_rot")
    net, feats, pts, cal, gout = _inputs(c)
    want = net.query_gradient(feats, pts, calibs=cal, grad_output=gout, precision="tc")
    view = pts[0].t().contiguous().t()[None]
    assert view.stride(2) == 3
    got = net.query_gradient(feats, view, calibs=cal, grad_output=gout, precision="tc")
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    v0, d0 = net.query_gradient(feats, pts[:, :, :0], calibs=cal, precision="tc")
    assert v0.shape == (1, 3, 0) and d0.shape == (1, 3, 0)
    with pytest.raises(ValueError):
        net.query_gradient(feats, pts, calibs=cal, precision="fp16")
    g = load_grad_case("g_nocalib")
    netg = build_net(g)
    feat = torch.cat([g["feat"], g["feat"]], 0).cuda()
    fh = netg.batch_feature_handle(feat)
    p = g["points"][0].cuda().contiguous()
    dp = torch.empty(3, p.shape[1], device="cuda")
    lib = _lib.load()
    for mode in (_lib.MODE_FP32, _lib.MODE_TC, _lib.MODE_AUTO):
        rc = lib.mp_query_points_grad_mode(netg.surface_classifier.handle(), fh.ptr, ctypes.c_void_p(p.data_ptr()), p.shape[1],
                                           p.shape[1], 1, None, 0, ctypes.c_float(spec.Z_SCALE), None, 0, None, 0,
                                           ctypes.c_void_p(dp.data_ptr()), p.shape[1], None, mode, _lib.stream_ptr())
        assert rc == -1 and b"single-map" in lib.mp_last_error()


def test_device_count_limits_the_points():
    from monoport_b200 import _lib
    c = load_grad_case("g_rot")
    net, feats, pts, cal, _ = _inputs(c)
    n = pts.shape[2]
    want = net.query_gradient(feats, pts, calibs=cal, precision="tc")
    k = n // 2 + 3
    count = torch.tensor([k], dtype=torch.int32, device="cuda")
    out = torch.full((1, n), -7.0, device="cuda")
    dp = torch.full((3, n), -7.0, device="cuda")
    p = pts[0].contiguous()
    fh = net.feature_handle(feats[0][0])
    lib = _lib.load()
    rc = lib.mp_query_points_grad_mode(net.surface_classifier.handle(), fh.ptr, ctypes.c_void_p(p.data_ptr()), n, n, 1,
                                       _lib.calib12(cal), _lib.PROJ_ORTHOGONAL, ctypes.c_float(spec.Z_SCALE), None, 0, ctypes.c_void_p(out.data_ptr()),
                                       n, ctypes.c_void_p(dp.data_ptr()), n, ctypes.c_void_p(count.data_ptr()), _lib.MODE_TC,
                                       _lib.stream_ptr())
    assert rc == 0, lib.mp_last_error()
    torch.cuda.synchronize()
    assert torch.equal(out[:, :k], want[0][0][:, :k]) and torch.equal(dp[:, :k], want[1][0][:, :k])
    assert bool((out[:, k:] == -7).all()) and bool((dp[:, k:] == -7).all())


def test_surface_normals_tc_against_exact():
    """the normals of forward_vertices' visible vertices of the synthetic person at R = 257: the direction of the tensor-core
    normals against the exact ones (reported as a distribution; at most 1 degree for 99 % of the vertices)"""
    from monoport_b200.recon import forward_vertices, surface_normals
    Ws, bs = spec.make_weights(spec.G_CHANNELS, 3)
    Ws, bs, feat, _ = spec.heightfield_person(Ws, bs, spec.make_feat(256, 128, 128, 4, 0.5))
    net = build_net("G", Ws, bs)
    if not net.surface_classifier.tc_supported():
        pytest.skip("no tensor-core program on this device")
    feats, cal, R = [[feat.cuda()]], spec.scene_calib(20, 0).cuda(), 257
    net.precision = "auto"
    vol = net.query_grid(feats[-1][0], cal, R, torch.tensor([-1.0] * 3), torch.tensor([1.0] * 3))
    X, Y, Z, _ = forward_vertices(vol[None, None], "front")
    exact = surface_normals(net, feats, X, Y, Z, cal, resolution=R)
    for precision in ("tc", "auto"):
        got = surface_normals(net, feats, X, Y, Z, cal, resolution=R, precision=precision)
        ok = (exact.norm(dim=1) > 0) & (got.norm(dim=1) > 0)
        ang = torch.rad2deg(torch.acos((got[ok] * exact[ok]).sum(1).clamp(-1, 1)))
        q = torch.quantile(ang.double(), torch.tensor([0.5, 0.9, 0.99, 0.999], dtype=torch.float64, device=ang.device)).tolist()
        print("surface_normals %s vs fp32 over %d vertices: angle median %.4f, p90 %.4f, p99 %.4f, p99.9 %.4f, max %.4f deg"
              % (precision, int(ok.sum()), q[0], q[1], q[2], q[3], ang.max().item()))
        assert ok.double().mean().item() >= 0.99 and q[2] <= 1.0 and math.isfinite(q[3])


@pytest.mark.parametrize("mode", ["fp32", "tc_out_of_range"])
def test_exact_route_takes_the_device_count(mode):
    """the exact gradient kernel with a point count on the device: MP_MODE_FP32, and MP_MODE_TC on a frame above the
    head's feature limit (the tensor-core launch skips, the exact one runs) -- the first k points bit for bit precision
    "fp32", the rest untouched"""
    from monoport_b200 import _lib
    c = load_grad_case("g_rot")
    net, feats, pts, cal, _ = _inputs(c)
    n = pts.shape[2]
    want = net.query_gradient(feats, pts, calibs=cal, precision="fp32")
    if mode != "fp32":
        net.surface_classifier.tc_feature_limit = 0.25
        assert feats[0][0].abs().max().item() > 0.25
    k = n // 2 + 5
    count = torch.tensor([k], dtype=torch.int32, device="cuda")
    out = torch.full((1, n), -7.0, device="cuda")
    dp = torch.full((3, n), -7.0, device="cuda")
    p = pts[0].contiguous()
    fh = net.feature_handle(feats[0][0])
    lib = _lib.load()
    rc = lib.mp_query_points_grad_mode(net.surface_classifier.handle(), fh.ptr, ctypes.c_void_p(p.data_ptr()), n, n, 1,
                                       _lib.calib12(cal), _lib.PROJ_ORTHOGONAL, ctypes.c_float(spec.Z_SCALE), None, 0,
                                       ctypes.c_void_p(out.data_ptr()), n, ctypes.c_void_p(dp.data_ptr()), n,
                                       ctypes.c_void_p(count.data_ptr()), _lib.MODE_FP32 if mode == "fp32" else _lib.MODE_TC,
                                       _lib.stream_ptr())
    assert rc == 0, lib.mp_last_error()
    torch.cuda.synchronize()
    assert torch.equal(out[:, :k], want[0][0][:, :k]) and torch.equal(dp[:, :k], want[1][0][:, :k])
    assert bool((out[:, k:] == -7).all()) and bool((dp[:, k:] == -7).all())


def test_frame_graph_renders_analytic_normals():
    """FrameGraph(render_normals="gradient") in a two-lane ring with netC: every frame's normal image is, bit for bit, eager
    colorization(norm=surface_normals(..., precision="auto")) on its vertices -- across an empty frame and a frame above
    the geometry head's feature limit (differentiated by the exact kernel on the device)."""
    from monoport_b200.engine import Seg3dLossless, make_query_func
    from monoport_b200.pipeline import FrameGraph, FrameGraphRing
    from monoport_b200.recon import colorization, surface_normals
    Ws, bs = spec.make_weights(spec.G_CHANNELS, 3)
    base = spec.make_feat(256, 128, 128, 4, 0.5)
    feats = []
    for k in range(3):
        W2, b2, f, _ = spec.heightfield_person(Ws, bs, base * (1.0 + 0.1 * k), channel=0)
        feats.append(f.cuda())
    net = build_net("G", W2, b2)
    if not net.surface_classifier.tc_supported():
        pytest.skip("no tensor-core program on this device")
    amax = [f.abs().max().item() for f in feats]
    assert amax[2] > amax[1] > amax[0]
    net.surface_classifier.tc_feature_limit = amax[1]             # feats[2] is above it
    cal = spec.scene_calib(20, 33)
    b = np.array([[-1.0, -1.0, -1.0]], dtype=np.float32)
    eng = Seg3dLossless(make_query_func(net), b, -b, [17, 33, 65], balance_value=0.5, faster=True).to("cuda")
    Wc, bc = spec.make_weights(spec.C_CHANNELS, 21)
    netC = build_net("C", Wc, bc)
    empty = feats[0].clone()
    empty[0, 0] = -5.0
    c0 = spec.make_feat(512, 128, 128, 22, 0.5).cuda()
    frames = [(feats[0], c0), (feats[1], c0), (empty, c0), (feats[2], c0), (feats[0], c0)]
    with pytest.raises(ValueError):
        FrameGraph(net, eng, cal, "front", with_encoder=False, render_normals="finite")
    ring = FrameGraphRing(lambda: FrameGraph(net, eng, cal, "front", with_encoder=False, netC=netC,
                                             render_normals="gradient"), n_lanes=2)
    n_out, calg = 0, cal.cuda()
    for (f, _), out in zip(frames, ring.run(iter(frames))):
        n_out += 1
        sdf, X, Y, Z, N, rnorm, rtex = out
        if sdf is None:
            assert f is empty and rnorm is None and rtex is None
            continue
        nrm = surface_normals(net, [[f]], X, Y, Z, calg, resolution=65, precision="auto")
        assert torch.equal(rnorm, colorization(None, None, X, Y, Z, calg, norm=nrm, resolution=65))
        ok = (nrm.norm(dim=1) > 0) & torch.isfinite(N).all(1)
        assert ok.double().mean().item() >= 0.99 and (nrm[ok] * N[ok]).sum(1).mean().item() >= 0.9
    assert n_out == len(frames)
    ring.close()
