"""GPU tests of the batched query(): B images in one launch (mp_query_points_batch) against the reference's batched goldens,
against B = 1 queries of each image, the per-image range guard, and the single-map entry points refusing a
batch handle.  Tolerances as in test_query_gpu.py."""
import ctypes

import pytest
import torch

from oracle import spec
from helpers import build_net
from batch_cases import batch_cases, load_batch_case

pytestmark = pytest.mark.gpu

TOL = {"fp32": 2e-5, "tc": 1e-4, "auto": 1e-4}
TOL_COLOUR = {"fp32": 2e-5, "tc": 1e-4, "auto": 1e-4}


def _modes(net):
    return ["fp32", "tc", "auto"] if net.surface_classifier.tc_supported() else ["fp32"]


def _single(net, feat, pts, cal, b):
    return net.query([[feat[b:b + 1]]], pts[b:b + 1], calibs=None if cal is None else cal[b:b + 1])[0][0]


@pytest.mark.parametrize("name", batch_cases())
def test_batched_query_matches_batched_reference_golden(name):
    c = load_batch_case(name)
    net = build_net(c)
    feat, pts = c["feat"].cuda(), c["points"].cuda()
    cal = c["calib"].cuda() if c["calib"] is not None else None
    for mode in _modes(net):
        net.precision = mode
        out = net.query([[torch.zeros_like(feat)]] * 3 + [[feat]], pts, calibs=cal)
        assert isinstance(out, list) and len(out) == 1 and out[0].shape == c["expected"].shape
        got = out[0].cpu()
        err = (got - c["expected"]).abs().max().item()
        tol = TOL_COLOUR if c["net"] == "C" else TOL
        assert err <= tol[mode], (name, mode, err)
        zero = c["expected"] == 0
        assert torch.equal(got[zero], c["expected"][zero]), "out-of-image points must be exactly 0"


def _five_images():
    c = load_batch_case("g_rot")
    extra = [spec.make_feat(256, 128, 128, 900 + k) for k in range(2)]
    feat = torch.cat([c["feat"]] + extra, 0)
    pts = torch.cat([c["points"], spec.make_points(1000, 901), spec.make_points(1000, 902)], 0)
    cal = torch.cat([c["calib"], spec.scene_calib(-30, 10), spec.scene_calib(45, 60)], 0)
    return c, feat, pts, cal


@pytest.mark.parametrize("B", [2, 5])
def test_batched_images_equal_single_queries(B):
    c, feat, pts, cal = _five_images()
    net = build_net(c)
    feat, pts, cal = feat[:B].cuda(), pts[:B].cuda(), cal[:B].cuda()
    for mode in _modes(net):
        net.precision = mode
        for n in (1, 63, 64, 65, 1000):
            p = pts[:, :, :n].contiguous()
            singles = [_single(net, feat, p, cal, b) for b in range(B)]
            for calib in (cal, cal[:, :3, :]):
                a = net.query([[feat]], p, calibs=calib)[0]
                assert a.shape == (B, 1, n)
                # permuted [B,N,3] view (RTL/main.py:176-177 layout)
                b_ = net.query([[feat]], p.permute(0, 2, 1).contiguous().permute(0, 2, 1), calibs=calib)[0]
                assert torch.equal(a, b_), (mode, n)
                for b in range(B):
                    assert torch.equal(a[b], singles[b]), (mode, n, b, (a[b] - singles[b]).abs().max().item())
        e = net.query([[feat]], torch.zeros(B, 3, 0, device="cuda"), calibs=cal)[0]
        assert e.shape == (B, 1, 0)


def test_batched_colour_head_equals_single_queries():
    c = load_batch_case("c_rot")
    net = build_net(c)
    feat, pts, cal = c["feat"].cuda(), c["points"].cuda(), c["calib"].cuda()
    for mode in _modes(net):
        net.precision = mode
        a = net.query([[feat]], pts, calibs=cal)[0]
        for b in range(c["B"]):
            one = _single(net, feat, pts, cal, b)
            assert torch.equal(a[b], one), (mode, b, (a[b] - one).abs().max().item())


def test_per_image_range_guard():
    """g_mixed: image 1 is above the geometry head's limit.  In "auto" mode it is evaluated by the exact kernel (equal to
    its fp32-mode single query, bit for bit), the others on the tensor cores (their tc-mode single queries, bit for bit)."""
    c = load_batch_case("g_mixed")
    net = build_net(c)
    if not net.surface_classifier.tc_supported():
        pytest.skip("no tensor-core program on this device")
    feat, pts, cal = c["feat"].cuda(), c["points"].cuda(), c["calib"].cuda()
    net.precision = "auto"
    got = net.query([[feat]], pts, calibs=cal)[0]
    net.precision = "fp32"
    exact1 = _single(net, feat, pts, cal, 1)
    net.precision = "tc"
    tc0, tc2 = _single(net, feat, pts, cal, 0), _single(net, feat, pts, cal, 2)
    assert torch.equal(got[1], exact1)
    assert torch.equal(got[0], tc0) and torch.equal(got[2], tc2)
    net.precision = "fp32"
    assert not torch.equal(got[0], _single(net, feat, pts, cal, 0)), "image 0 is in range: the tensor cores evaluate it"
    assert (got.cpu() - c["expected"]).abs().max().item() <= TOL["auto"]


def test_channels_last_batch_bound_in_place_equals_contiguous_upload():
    c = load_batch_case("g_rot")
    net = build_net(c)
    feat, pts, cal = c["feat"].cuda(), c["points"].cuda(), c["calib"].cuda()
    feat_cl = feat.contiguous(memory_format=torch.channels_last)
    assert not feat_cl.is_contiguous() and torch.equal(feat_cl, feat)
    for mode in _modes(net):
        net.precision = mode
        a = net.query([[feat]], pts, calibs=cal)[0].clone()
        b = net.query([[feat_cl]], pts, calibs=cal)[0]
        assert torch.equal(a, b), mode


def test_forward_with_labels_batch_of_two():
    """forward(images, points, calibs, labels) with B = 2: the PyTorch encoder, the batched query, the loss -- against the
    oracle evaluated per image on the same encoder features."""
    c = load_batch_case("g_rot")
    net = build_net(c)
    net.image_filter.cuda().eval()
    net.precision = "fp32"
    g = torch.Generator().manual_seed(3)
    images = torch.rand(2, 3, 512, 512, generator=g).cuda()
    pts, cal = c["points"][:2].cuda(), c["calib"][:2].cuda()
    labels = torch.rand(2, 1, pts.shape[2], generator=g).cuda()
    pred, loss = net(images, pts, cal, labels=labels)
    assert pred.shape == (2, 1, pts.shape[2])
    with torch.no_grad():
        feats = net.filter(images)[-1][0].cpu()
    want = torch.stack([spec.query_ref(feats[b], c["points"][b], c["calib"][b], c["Ws"], c["bs"], spec.LAST_SIGMOID)
                        for b in range(2)])
    assert (pred.cpu() - want).abs().max().item() <= TOL["fp32"]
    want_loss = torch.nn.functional.mse_loss(want, labels.cpu())
    assert abs(loss.item() - want_loss.item()) <= 1e-6


def test_mismatched_batch_sizes_raise_value_error():
    c = load_batch_case("g_rot")
    net = build_net(c)
    feat, pts, cal = c["feat"].cuda(), c["points"].cuda(), c["calib"].cuda()
    with pytest.raises(ValueError):
        net.query([[feat]], pts[:2], calibs=cal)
    with pytest.raises(ValueError):
        net.query([[feat]], pts, calibs=cal[:2])
    with pytest.raises(ValueError):
        net.query([[feat[:1]]], pts, calibs=cal[:1])
    with pytest.raises(ValueError):
        net.query([[feat[:1]]], pts[:1], calibs=cal)
    with pytest.raises(ValueError):
        net.feature_handle(feat)                    # the single-map handle keeps refusing batches


def test_single_map_entry_points_refuse_a_batch_handle():
    from monoport_b200 import _lib
    from monoport_b200.engine import Seg3dLossless, make_query_func
    from monoport_b200.recon import colorization
    import numpy as np
    c = load_batch_case("g_rot")
    net = build_net(c)
    lib = _lib.load()
    feat, cal = c["feat"].cuda(), c["calib"].cuda()
    fh = net.batch_feature_handle(feat)
    head = net.surface_classifier.handle()
    st = _lib.stream_ptr(torch.device("cuda:0"))
    z = ctypes.c_float(spec.Z_SCALE)
    c12 = _lib.calib12(c["calib"][:1])
    lo, hi = _lib.f3((-1, -1, -1)), _lib.f3((1, 1, 1))
    out = torch.empty(3 * 9 ** 3, device="cuda")
    pts = c["points"][0].contiguous().cuda()
    optr = ctypes.c_void_p(out.data_ptr())
    peers = (ctypes.c_void_p * 1)(out.data_ptr())
    calls = {
        "points": lambda: lib.mp_query_points(head, fh.ptr, ctypes.c_void_p(pts.data_ptr()), 8, pts.shape[1], 1, c12, 0, z, optr,
                                              8, _lib.MODE_FP32, st),
        "grid": lambda: lib.mp_query_grid(head, fh.ptr, 9, 0, 9, lo, hi, c12, 0, z, optr, _lib.MODE_FP32, st),
        "grid_range": lambda: lib.mp_query_grid_range(head, fh.ptr, 9, 0, 100, lo, hi, c12, 0, z, optr, _lib.MODE_FP32, st),
        "peers": lambda: lib.mp_query_grid_peers(head, fh.ptr, 9, 0, 9, lo, hi, c12, 0, z, peers, 1, _lib.MODE_FP32, st),
        "host": lambda: lib.mp_query_points_host(head, fh.ptr, None, None, 0, c12, 0, z, None, _lib.MODE_FP32, st),
        "grid_host": lambda: lib.mp_query_grid_host(head, fh.ptr, None, 9, 0, 0, lo, hi, c12, 0, z, None, _lib.MODE_FP32, st),
    }
    oc = ctypes.c_void_p()
    _lib.check(lib.mp_octree_create(2, (ctypes.c_int * 2)(5, 9), lo, hi, ctypes.c_float(0.5), 1, None, ctypes.byref(oc)))
    ne = ctypes.c_int(0)
    calls["octree"] = lambda: lib.mp_octree_run_fused(oc, head, fh.ptr, c12, 0, z, _lib.MODE_FP32, optr, ctypes.byref(ne), None, st)
    calls["octree_async"] = lambda: lib.mp_octree_run_fused_async(oc, head, fh.ptr, c12, 0, z, _lib.MODE_FP32, optr, st)
    calls["colorize"] = lambda: lib.mp_colorize_surface(head, fh.ptr, optr, optr, optr, 4, 9, lo, hi, c12, 0, z, optr, st)
    for what, call in calls.items():
        assert call() == -1, what
        assert b"single-map" in lib.mp_last_error(), what
    lib.mp_octree_destroy(oc)
    # the Python layers: grid query with the batch handle, the occupancy engine and colourisation with batched features
    with pytest.raises(RuntimeError, match="single-map"):
        net.query_grid(feat[:1], cal[:1], 9, (-1, -1, -1), (1, 1, 1), fh=fh)
    b = np.array([[-1.0, -1.0, -1.0]], dtype=np.float32)
    eng = Seg3dLossless(make_query_func(net), b, -b, [5, 9], balance_value=0.5, faster=True).to("cuda")
    with pytest.raises(ValueError):
        eng(im_feat_list=[[feat]], calib_tensor=cal)
    cc = load_batch_case("c_rot")
    netC = build_net(cc)
    X = torch.zeros(4, dtype=torch.int64, device="cuda")
    with pytest.raises(ValueError):
        colorization(netC, [[cc["feat"].cuda()]], X, X, X.float(), cc["calib"].cuda(), resolution=9)
