"""The dense grid query of a Sigmoid head on the tensor cores evaluates only the nodes that project into the image and stores
+0 for the others (DESIGN.md §F1).  Its volume must be the dense program's bit for bit: the same values as query() of the
node centres through point rows, compared as int32 views so that the sign of zero and NaN payloads count.  Heads whose
value outside the image is not always +0 (Tanh) keep the dense launch; out-of-range frames go to the exact kernel; a
map with a NaN keeps every node in the list."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import spec
from helpers import build_net
from head_cases import build_head_net

pytestmark = pytest.mark.gpu

BOX = ((-1.0, -1.0, -1.0), (1.0, 1.0, 1.0))


def _bits(t):
    return t.contiguous().view(torch.int32).cpu()


def _node_centres(R, lin0=0, n=None):
    """world points of nodes [lin0, lin0 + n) in z-major order, rounded op by op as the kernels' grid source rounds them"""
    n = R ** 3 - lin0 if n is None else n
    lin = np.arange(lin0, lin0 + n, dtype=np.int64)
    c = np.stack([lin % R, (lin // R) % R, lin // (R * R)]).astype(np.float32)
    lo = np.array(BOX[0], dtype=np.float32)[:, None]
    ext = np.array(BOX[1], dtype=np.float32)[:, None] - lo
    half = np.float32(1.0 / (2.0 * R))
    return torch.from_numpy(((c / np.float32(R) + half) * ext + lo).astype(np.float32))


def _rows_query(net, feat, cal, R, lin0=0, n=None):
    pts = _node_centres(R, lin0, n)
    return net.query([[feat]], pts[None].cuda(), calibs=cal.cuda())[0][0, 0]


@pytest.fixture(scope="module")
def bench_case():
    import bench
    _, Ws, bs, feats = bench.synthetic(n_feat=1)
    net = build_net("G", Ws, bs)
    if not net.surface_classifier.tc_supported():
        pytest.skip("no tensor-core program on this device")
    net.precision = "tc"
    return net, Ws, bs, feats[0].cuda(), bench.scene_calib()


@pytest.mark.parametrize("R", [65, 257])
def test_grid_equals_rows_query(bench_case, R):
    net, _, _, feat, cal = bench_case
    vol = net.query_grid(feat, cal.cuda(), R, *BOX)
    want = _rows_query(net, feat, cal, R)
    assert torch.equal(_bits(vol).reshape(-1), _bits(want))
    outside = (vol == 0).float().mean().item()
    assert 0.05 < outside < 0.5, outside          # the bench camera: about 14 % of the nodes project outside the image


def test_slabs_ranges_and_host_entry_point(bench_case):
    from monoport_b200 import _lib
    net, _, _, feat, cal = bench_case
    R = 65
    vol = _bits(net.query_grid(feat, cal.cuda(), R, *BOX)).reshape(-1)
    for z0, nz in ((0, 1), (3, 17), (40, 25)):
        slab = net.query_grid(feat, cal.cuda(), R, *BOX, z0=z0, nz=nz)
        assert torch.equal(_bits(slab).reshape(-1), vol[z0 * R * R:(z0 + nz) * R * R]), (z0, nz)
    for lin0, n in ((1234, 4321), (R * R - 7, 2 * R * R + 11), (5, R ** 3 - 9)):      # ranges that start and end inside planes
        part = net.query_grid_range(feat, cal.cuda(), R, *BOX, lin0=lin0, n=n)
        assert torch.equal(_bits(part), vol[lin0:lin0 + n]), (lin0, n)
    lib = _lib.load()
    feat_host = feat.cpu().contiguous()
    for R_h, z0, nz in ((65, 0, 65), (165, 7, 150)):
        want = _bits(net.query_grid(feat, cal.cuda(), R_h, *BOX, z0=z0, nz=nz))
        fh = ctypes.c_void_p()
        _lib.check(lib.mp_feat_create(256, feat.shape[2], feat.shape[3], ctypes.byref(fh)))
        out = torch.full((nz, R_h, R_h), float("nan"), dtype=torch.float32).pin_memory()
        _lib.check(lib.mp_query_grid_host(net.surface_classifier.handle(), fh, ctypes.c_void_p(feat_host.data_ptr()), R_h, z0, nz,
                                          _lib.f3(BOX[0]), _lib.f3(BOX[1]), _lib.calib12(cal), 0, ctypes.c_float(spec.Z_SCALE),
                                          ctypes.c_void_p(out.data_ptr()), _lib.MODE_TC, _lib.stream_ptr(torch.device("cuda:0"))))
        lib.mp_feat_destroy(fh)
        assert torch.equal(_bits(out), want), (R_h, z0, nz)


def test_single_gpu_peer_form(bench_case):
    """mp_query_grid_range_peers with one peer volume (the own one): the range's nodes, listed or zero, land at their node
    index of the full volume, and nothing outside the range is touched"""
    from monoport_b200 import _lib
    net, _, _, feat, cal = bench_case
    R = 65
    vol = _bits(net.query_grid(feat, cal.cuda(), R, *BOX)).reshape(-1)
    lib = _lib.load()
    for lin0, n in ((0, R ** 3), (R * R + 3, 20000)):
        peer = torch.full((R ** 3,), float("nan"), dtype=torch.float32, device="cuda")
        ptrs = (ctypes.c_void_p * 1)(peer.data_ptr())
        fh = net.feature_handle(feat)
        _lib.check(lib.mp_query_grid_range_peers(net.surface_classifier.handle(), fh.ptr, R, lin0, n, _lib.f3(BOX[0]),
                                                 _lib.f3(BOX[1]), _lib.calib12(cal), _lib.PROJ_ORTHOGONAL,
                                                 ctypes.c_float(net.normalizer.scale), ptrs, 1, net._mode(),
                                                 _lib.stream_ptr(feat.device)))
        torch.cuda.synchronize()
        got = _bits(peer)
        assert torch.equal(got[lin0:lin0 + n], vol[lin0:lin0 + n]), (lin0, n)
        nan_bits = _bits(torch.tensor([float("nan")]))[0]
        assert bool((got[:lin0] == nan_bits).all()) and bool((got[lin0 + n:] == nan_bits).all()), (lin0, n)


def test_cameras_with_every_node_inside_and_outside(bench_case):
    net, _, _, feat, cal = bench_case
    R = 33
    inside = cal.clone()
    inside[0, :3, :] *= 0.25                      # the whole box projects into the image
    outside = cal.clone()
    outside[0, 0, 3] += 10.0                      # shifted far off the image
    for c, expect_zero in ((inside, False), (outside, True)):
        vol = net.query_grid(feat, c.cuda(), R, *BOX)
        assert torch.equal(_bits(vol).reshape(-1), _bits(_rows_query(net, feat, c, R)))
        assert bool((vol == 0).all()) == expect_zero
    assert bool((_bits(net.query_grid(feat, outside.cuda(), R, *BOX)) == 0).all())      # +0, not -0


def test_tanh_head_keeps_the_dense_launch(bench_case):
    """0 * tanh(logit) carries the logit's sign: a Tanh head's volume has -0 outside the image, as the dense launch gives"""
    _, Ws, bs, feat, cal = bench_case
    net = build_head_net(dict(chans=[257, 1024, 512, 256, 128, 1], last_op=spec.LAST_TANH, Ws=Ws, bs=bs, proj="orthogonal"))
    if not net.surface_classifier.tc_supported():
        pytest.skip("no tensor-core program for this head")
    net.precision = "tc"
    R = 65
    vol = net.query_grid(feat, cal.cuda(), R, *BOX)
    got = _bits(vol).reshape(-1)
    assert torch.equal(got, _bits(_rows_query(net, feat, cal, R)))
    neg_zero = _bits(torch.tensor([-0.0]))[0]
    assert bool((got == neg_zero).any())


def test_out_of_range_frame_equals_the_exact_kernel(bench_case):
    net, _, _, feat, cal = bench_case
    big = feat * 40.0
    assert big.abs().max().item() > 12.0          # the default feature limit of a Sigmoid head
    R = 65
    net.precision = "fp32"
    exact = _bits(net.query_grid(big, cal.cuda(), R, *BOX))
    try:
        for mode in ("auto", "tc"):
            net.precision = mode
            assert torch.equal(_bits(net.query_grid(big, cal.cuda(), R, *BOX)), exact), mode
    finally:
        net.precision = "tc"


def test_map_with_a_nan_keeps_every_node(bench_case):
    """the guard's maximum ignores a NaN, and 0 * NaN is NaN: every node is evaluated, as the dense launch does"""
    net, _, _, feat, cal = bench_case
    bad = feat.clone()
    bad[0, 3, :, -1] = float("nan")               # a column at the image's edge, which nodes just outside it sample too
    R = 65
    vol = net.query_grid(bad, cal.cuda(), R, *BOX)
    assert torch.equal(_bits(vol).reshape(-1), _bits(_rows_query(net, bad, cal, R)))
    assert bool(torch.isnan(vol).any())
