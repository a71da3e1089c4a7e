"""The demo's two images inside the captured frame step (FrameGraph(netC=..., render_normals=True)): the enqueue-only surface
render mp_colorize_surface_async against the eager colorization() in and out of the colour program's validated range, the
normal image, FrameGraphRing frame sequences, both encoders under capture, and the refusals of the new entry points.  A
capture that succeeds is itself the check that the step never synchronises with the host."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import spec
from helpers import build_net

pytestmark = pytest.mark.gpu

B_MIN, B_MAX = (-1.0, -1.0, -1.0), (1.0, 1.0, 1.0)


def _colour_net():
    Wc, bc = spec.make_weights(spec.C_CHANNELS, 21)
    return build_net("C", Wc, bc), Wc, bc


def _vertices(R=65):
    from monoport_b200.recon import forward_vertices
    vol = torch.from_numpy(spec.analytic_volume(R, "ellipsoid"))[None, None].cuda()
    X, Y, Z, _ = forward_vertices(vol, "front")
    return X, Y, Z


def _render_async(netC, featc, X, Y, Z, cal, R, mode, canvas=None):
    """mp_colorize_surface_async on buffers of capacity R*R whose tail past the count holds vertex (0, 0): the count is only
    known on the device"""
    from monoport_b200 import _lib
    from monoport_b200.modeling.geometry import perspective
    k, cap = X.numel(), R * R
    Xb = torch.zeros(cap, dtype=torch.int64, device="cuda")
    Yb = torch.zeros(cap, dtype=torch.int64, device="cuda")
    Zb = torch.zeros(cap, dtype=torch.float32, device="cuda")
    Xb[:k], Yb[:k], Zb[:k] = X, Y, Z
    count = torch.tensor([k], dtype=torch.int64, device="cuda")
    img = torch.ones((R, R, 3), dtype=torch.float32, device="cuda") if canvas is None else canvas.clone()
    fh = netC.feature_handle(featc)
    proj = _lib.PROJ_PERSPECTIVE if netC.projection is perspective else _lib.PROJ_ORTHOGONAL
    _lib.check(_lib.load().mp_colorize_surface_async(
        netC.surface_classifier.handle(), fh.ptr, ctypes.c_void_p(Xb.data_ptr()), ctypes.c_void_p(Yb.data_ptr()),
        ctypes.c_void_p(Zb.data_ptr()), ctypes.c_void_p(count.data_ptr()), cap, R, _lib.f3(B_MIN), _lib.f3(B_MAX),
        _lib.calib12(cal), proj, ctypes.c_float(netC.normalizer.scale), mode, ctypes.c_void_p(img.data_ptr()),
        _lib.stream_ptr()), "mp_colorize_surface_async")
    torch.cuda.synchronize()
    return img


def test_async_render_in_range_equals_eager():
    """AUTO, a frame inside the colour program's range: the same tensor-core kernel on the same vertices as the eager
    mp_colorize_surface, bit for bit -- the device-side count and the device-side guard change nothing."""
    from monoport_b200 import _lib
    from monoport_b200.recon import colorization
    netC, _, _ = _colour_net()
    assert netC.surface_classifier.tc_supported()
    featc = spec.make_feat(512, 128, 128, 22).cuda()
    cal = spec.scene_calib(20, 33).cuda()
    X, Y, Z = _vertices()
    eager = colorization(netC, [[featc]], X, Y, Z, cal, resolution=65)
    got = _render_async(netC, featc, X, Y, Z, cal, 65, _lib.MODE_AUTO)
    assert torch.equal(got, eager)


@pytest.mark.parametrize("precision", ["auto", "fp32"])
def test_async_render_out_of_range_is_the_exact_route(precision):
    """A frame above the head's limit (forced low) is rendered by the exact twin on the device: within the fp32 bar of the
    restatement, and bit for bit what eager colorization() gives through netC.query's exact kernel.  The same with
    precision="fp32", where the exact kernel is the only launch."""
    from monoport_b200.recon import colorization
    netC, Wc, bc = _colour_net()
    netC.precision = precision
    netC.surface_classifier.tc_feature_limit = 0.5
    featc = spec.make_feat(512, 128, 128, 22)
    cal = spec.scene_calib(20, 33)
    X, Y, Z = _vertices()
    assert featc.abs().max().item() > 0.5
    eager = colorization(netC, [[featc.cuda()]], X, Y, Z, cal.cuda(), resolution=65)
    got = _render_async(netC, featc.cuda(), X, Y, Z, cal.cuda(), 65, netC._mode())

    def qc(points, calib):
        return spec.query_ref(featc, points, calib, Wc, bc, spec.LAST_TANH)
    want = spec.colorization_ref(qc, X.cpu(), Y.cpu(), Z.cpu(), cal, resolution=65)
    err = (got.cpu() - want).abs().max().item()
    diff = (got != eager).any(-1).nonzero()
    print("out of range [%s]: max|async - restatement| = %.3e, pixels differing from eager: %d" % (precision, err, len(diff)))
    assert err <= 2e-5
    assert torch.equal(got, eager), diff[:10].tolist()


def _graph_setup():
    from monoport_b200.engine import Seg3dLossless, make_query_func
    Ws, bs = spec.make_weights(spec.G_CHANNELS, 3)
    base = spec.make_feat(256, 128, 128, 4, 0.5)
    feats = []
    for k in range(3):
        W2, b2, f, _ = spec.heightfield_person(Ws, bs, base * (1.0 + 0.1 * k), channel=0)
        feats.append(f.cuda())
    net = build_net("G", W2, b2)
    cal = spec.scene_calib(20, 33)
    b = np.array([[-1.0, -1.0, -1.0]], dtype=np.float32)
    eng = Seg3dLossless(make_query_func(net), b, -b, [17, 33, 65], balance_value=0.5, faster=True).to("cuda")
    return net, eng, cal, feats


def test_frame_graph_ring_renders_the_demo_frame():
    """Two lanes with netC and the normal image, features given: every frame's result() is the geometry-only graph's,
    and rendered() is eager colorization(norm=N) and colorization(netC, ...) on that frame's vertices -- across an empty
    frame and a colour frame outside the tensor-core program's range (rendered by the exact twin) between in-range ones."""
    from monoport_b200.pipeline import FrameGraph, FrameGraphRing
    from monoport_b200.recon import colorization
    net, eng, cal, feats = _graph_setup()
    netC, _, _ = _colour_net()
    empty = feats[0].clone()
    empty[0, 0] = -5.0
    c0 = spec.make_feat(512, 128, 128, 22, 0.5).cuda()
    c1 = spec.make_feat(512, 128, 128, 23, 0.5).cuda()
    big = c0 * 60.0                                       # far above the colour head's limit of 8
    frames = [(feats[0], c0), (feats[1], c1), (empty, c0), (feats[2], big), (feats[0], c1)]
    plain = FrameGraphRing(lambda: FrameGraph(net, eng, cal, "front", with_encoder=False), n_lanes=2)
    want = [tuple(None if t is None else t.clone() for t in out) for out in plain.run(f for f, _ in frames)]
    plain.close()
    ring = FrameGraphRing(lambda: FrameGraph(net, eng, cal, "front", with_encoder=False, netC=netC, render_normals=True),
                          n_lanes=2)
    n_out = 0
    for (f, c), w, out in zip(frames, want, ring.run(iter(frames))):
        n_out += 1
        assert len(out) == 7
        sdf, X, Y, Z, N, rnorm, rtex = out
        if w[0] is None:
            assert sdf is None and rnorm is None and rtex is None
            continue
        for a, b in zip(w, (sdf, X, Y, Z, N)):
            assert torch.equal(a, b)
        assert torch.equal(rnorm, colorization(netC, None, X, Y, Z, cal.cuda(), norm=N, resolution=65))
        eager = colorization(netC, [[c]], X, Y, Z, cal.cuda(), resolution=65, b_min=B_MIN, b_max=B_MAX)
        assert torch.equal(rtex, eager), (rtex != eager).any(-1).nonzero()[:10].tolist()
    assert n_out == len(frames)
    ring.close()


def test_frame_graph_renders_with_both_encoders_under_capture():
    """HG encoder for netG and ResBlk encoder for netC (with netG's map as its prior) inside the captured step.  The set
    pixels are exactly those of the frame's visible vertices; the colours agree with an eager colorization of the eager
    encoders' map on those vertices to 1e-3: cudnn may pick other convolution algorithms under capture, so the encoder
    outputs differ by float noise, which the colour head carries into its output (the existing geometry test allows the
    same noise as a few mask nodes)."""
    from monoport_b200.pipeline import FrameGraph
    from monoport_b200.recon import colorization, forward_vertices
    net, eng, cal, feats = _graph_setup()
    netC, _, _ = _colour_net()
    net.image_filter.cuda()
    netC.image_filter.cuda()
    img = (torch.rand(1, 3, 512, 512, generator=torch.Generator().manual_seed(5)) * 2 - 1).cuda()
    imgc = (torch.rand(1, 3, 512, 512, generator=torch.Generator().manual_seed(6)) * 2 - 1).cuda()

    def hook(f):
        f = f.clone()
        f[:, 0] = feats[0][:, 0]
        return f
    with torch.no_grad():
        fe = hook(net.filter(img)[-1][0])
        featc = netC.filter(imgc, feat_prior=fe)[-1][0]
        sdf = eng(im_feat_list=[[fe]], calib_tensor=cal.cuda())
        Xe, Ye, _, _ = forward_vertices(sdf, "front")
    fg = FrameGraph(net, eng, cal, "front", with_encoder=True, feature_hook=hook, netC=netC, render_normals=True)
    for _ in range(2):
        sdf_g, X, Y, Z, N = fg.launch(img, imgc).result()
        rnorm, rtex = fg.rendered()
        assert sdf_g is not None and rnorm is not None and rtex is not None
        eager = colorization(netC, [[featc]], X, Y, Z, cal.cuda(), resolution=65)
        set_g, set_e = (rtex != 1.0).any(-1), (eager != 1.0).any(-1)
        assert torch.equal(set_g, set_e)
        cols_g = set(zip(X.tolist(), Y.tolist()))
        assert len(cols_g ^ set(zip(Xe.tolist(), Ye.tolist()))) <= 64
        err = (rtex - eager).abs().max().item()
        print("captured encoders: max|graph - eager| over the colour image = %.3e" % err)
        assert err <= 1e-3
        assert torch.equal(rnorm, colorization(netC, None, X, Y, Z, cal.cuda(), norm=N, resolution=65))
    fg.close()


def test_new_entry_points_refuse_bad_arguments():
    """A batch handle, a 1-channel head and bad counts / capacities are refused (MP_E_INVALID) before anything is enqueued."""
    from monoport_b200 import _lib
    from monoport_b200.modeling.MonoPortNet import FeatureHandle
    lib = _lib.load()
    netC, _, _ = _colour_net()
    netG = build_net("G", *spec.make_weights(spec.G_CHANNELS, 3))
    R, cap = 9, 81
    buf = torch.zeros(4 * cap, dtype=torch.int64, device="cuda")
    p = ctypes.c_void_p(buf.data_ptr())
    lo, hi, c12 = _lib.f3(B_MIN), _lib.f3(B_MAX), _lib.calib12(spec.scene_calib(20, 33))
    st = _lib.stream_ptr()
    fc = netC.feature_handle(spec.make_feat(512, 16, 16, 1).cuda())
    fg = netG.feature_handle(spec.make_feat(256, 16, 16, 1).cuda())
    fb = FeatureHandle(512, 16, 16, torch.device("cuda"), B=2)
    hc, hg = netC.surface_classifier.handle(), netG.surface_classifier.handle()

    def colour(head, fh, count=p, capacity=cap, r=R):
        return lib.mp_colorize_surface_async(head, fh.ptr, p, p, p, count, capacity, r, lo, hi, c12, 0, ctypes.c_float(1.28),
                                             _lib.MODE_AUTO, p, st)
    assert colour(hc, fc) == _lib.MP_OK
    assert colour(hc, fb) == -1                     # batch handle
    assert colour(hg, fg) == -1                     # 1-channel head
    assert colour(hc, fc, capacity=-1) == -1
    assert colour(hc, fc, capacity=R * R + 1) == -1
    assert colour(hc, fc, r=0) == -1
    assert colour(hc, fc, count=None) == -1
    assert lib.mp_render_normals_async(p, p, p, p, cap, R, p, st) == _lib.MP_OK
    assert lib.mp_render_normals_async(p, p, p, p, R * R + 1, R, p, st) == -1
    assert lib.mp_render_normals_async(p, p, p, p, -1, R, p, st) == -1
    assert lib.mp_render_normals_async(p, p, p, None, cap, R, p, st) == -1
    torch.cuda.synchronize()
