"""GPU tests of the batched point gradient (MonoPortNet.query_gradient on [B,C,H,W] maps -> mp_query_points_grad_batch): the
reference's batched autograd goldens in every precision, image b against the B = 1 call on image b and the value against
batched query() bit for bit, the per-image range guard, capture in a CUDA graph, and the argument handling."""
import ctypes

import pytest
import torch

from oracle import spec
from helpers import build_net
from batch_grad_cases import BATCH_GRAD_CASES, load_batch_grad_case, single
from grad_cases import tc_bar, within_bar
from shape_cases import load_shape_case

pytestmark = pytest.mark.gpu

PRECISIONS = ["fp32", "tc", "auto"]


def _inputs(c, precision="fp32"):
    net = build_net(c)
    if precision != "fp32" and not net.surface_classifier.tc_supported():
        pytest.skip("no tensor-core program on this device")
    gout = c["grad_output"].cuda() if c.get("grad_output") is not None else None
    cal = c["calib"].cuda() if c["calib"] is not None else None
    return net, [[c["feat"].cuda()]], c["points"].cuda(), cal, gout


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", BATCH_GRAD_CASES)
def test_batch_gradient_matches_reference_golden(name, precision):
    c = load_batch_grad_case(name)
    net, feats, pts, cal, gout = _inputs(c, precision)
    val, dp = net.query_gradient(feats, pts, calibs=cal, grad_output=gout, precision=precision)
    B, N = pts.shape[0], pts.shape[2]
    assert val.shape == (B, c["chans"][-1], N) and dp.shape == (B, 3, N)
    val, dp = val.cpu(), dp.cpu()
    outside = (c["value"] == 0).all(1)
    for b in range(B):
        # (g_mixed image 1 is above the geometry head's limit: "tc" and "auto" differentiate it exactly)
        exact = precision == "fp32" or (name == "g_mixed" and b == 1)
        assert (val[b] - c["value"][b]).abs().max().item() <= (2e-5 if exact else 1e-4), b
        ok, msg = within_bar(dp[b], c["grad32"][b]) if precision == "fp32" else tc_bar(dp[b], c["grad64"][b])
        print(name, precision, b, msg)
        assert ok, (b, msg)
        assert bool((dp[b][:, outside[b]] == 0).all()), b


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", BATCH_GRAD_CASES)
def test_batch_equals_single_calls_and_batched_query_bit_for_bit(name, precision):
    """image b of the batched call == the B = 1 call on image b (value and d points); the batched value == batched query()
    in the same precision"""
    c = load_batch_grad_case(name)
    net, feats, pts, cal, gout = _inputs(c, precision)
    val, dp = net.query_gradient(feats, pts, calibs=cal, grad_output=gout, precision=precision)
    for b in range(c["B"]):
        s = single(c, b)
        _, f1, p1, c1, g1 = _inputs(s, precision)
        v1, d1 = net.query_gradient(f1, p1, calibs=c1, grad_output=g1, precision=precision)
        assert torch.equal(val[b:b + 1], v1) and torch.equal(dp[b:b + 1], d1), b
    net.precision = precision
    assert torch.equal(val, net.query(feats, pts, calibs=cal)[0])


def test_mixed_batch_takes_the_exact_kernel_for_the_image_above_the_limit():
    """g_mixed, image 1 above the geometry head's limit: under "tc" and "auto" it has its "fp32" bits, images 0 and 2 have
    their "tc" bits (the B = 1 tensor-core program on each)"""
    c = load_batch_grad_case("g_mixed")
    net, feats, pts, cal, _ = _inputs(c, "tc")
    exact = net.query_gradient(feats, pts, calibs=cal, precision="fp32")
    for precision in ("tc", "auto"):
        got = net.query_gradient(feats, pts, calibs=cal, precision=precision)
        assert torch.equal(got[0][1], exact[0][1]) and torch.equal(got[1][1], exact[1][1]), precision
        for b in (0, 2):
            s = single(c, b)
            _, f1, p1, c1, _ = _inputs(s, "tc")
            one = net.query_gradient(f1, p1, calibs=c1, precision="tc")
            assert torch.equal(got[0][b], one[0][0]) and torch.equal(got[1][b], one[1][0]), (precision, b)
            assert not torch.equal(got[1][b], exact[1][b]), (precision, b)


@pytest.mark.parametrize("precision", ["fp32", "tc"])
def test_batched_call_is_captured_in_a_cuda_graph(precision):
    """the batched call enqueues only (calibs on the device, nothing read back): it records into a CUDA graph, and a replay
    on new points gives what an eager call on them gives"""
    c = load_batch_grad_case("g_rot")
    net, feats, pts, cal, _ = _inputs(c, precision)
    static_pts = pts.clone()
    net.query_gradient(feats, static_pts, calibs=cal, precision=precision)          # handle, upload, per-frame products
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        val, dp = net.query_gradient(feats, static_pts, calibs=cal, precision=precision)
    moved = pts.flip(2).contiguous()
    static_pts.copy_(moved)
    g.replay()
    torch.cuda.synchronize()
    want = net.query_gradient(feats, moved, calibs=cal, precision=precision)
    assert torch.equal(val, want[0]) and torch.equal(dp, want[1])


def test_batch_arguments_and_refusals():
    from monoport_b200 import _lib
    c = load_batch_grad_case("c_rot")
    net, feats, pts, cal, gout = _inputs(c)
    B, N = pts.shape[0], pts.shape[2]
    view = pts.transpose(1, 2).contiguous().transpose(1, 2)      # [B,3,N] views of [B,N,3] rows
    assert view.stride(2) == 3
    want = net.query_gradient(feats, pts, calibs=cal, grad_output=gout)
    got = net.query_gradient(feats, view, calibs=cal, grad_output=gout)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    ones = net.query_gradient(feats, pts, calibs=cal)
    ones2 = net.query_gradient(feats, pts, calibs=cal, grad_output=torch.ones(B, 3, N, device="cuda"))
    assert torch.equal(ones[0], ones2[0]) and torch.equal(ones[1], ones2[1])
    v0, d0 = net.query_gradient(feats, pts[:, :, :0], calibs=cal)
    assert v0.shape == (B, 3, 0) and d0.shape == (B, 3, 0)
    with pytest.raises(ValueError):
        net.query_gradient(feats, pts[:1], calibs=cal)                       # points of another B
    with pytest.raises(ValueError):
        net.query_gradient(feats, pts, calibs=cal[:1])                       # calibs of another B
    with pytest.raises(ValueError):
        net.query_gradient(feats, pts, calibs=cal, grad_output=gout[:1])
    with pytest.raises(ValueError):
        net.query_gradient(feats, pts, calibs=cal, grad_output=gout[:, :1])
    with pytest.raises(ValueError):
        net.query_gradient(feats, pts, calibs=cal, precision="fp16")
    with pytest.raises(NotImplementedError):
        net.train().query_gradient(feats, pts, calibs=cal)
    net.eval()
    with pytest.raises(RuntimeError):
        net.query_gradient([[c["feat"]]], pts, calibs=cal)
    # the C-ABI: B must be the handle's
    fh = net.batch_feature_handle(feats[0][0])
    p = pts.contiguous()
    dp = torch.empty(B, 3, N, device="cuda")
    lib = _lib.load()
    rc = lib.mp_query_points_grad_batch(net.surface_classifier.handle(), fh.ptr, B + 1, ctypes.c_void_p(p.data_ptr()), N,
                                        3 * N, N, 1, None, 0, ctypes.c_float(spec.Z_SCALE), None, None,
                                        ctypes.c_void_p(dp.data_ptr()), _lib.MODE_FP32, _lib.stream_ptr())
    assert rc == -1 and b"does not match" in lib.mp_last_error()


def test_batch_of_maps_above_65536_texels():
    c = load_shape_case("g_over")                     # 257 x 256
    net = build_net(c)
    if not net.surface_classifier.tc_supported():
        pytest.skip("no tensor-core program on this device")
    feat = torch.cat([c["feat"], c["feat"].flip(3) * 0.5], 0).cuda()
    pts = torch.cat([c["points"], c["points"].flip(2)], 0).cuda()
    cal = torch.cat([c["calib"], c["calib"]], 0).cuda() if c["calib"] is not None else None
    exact = net.query_gradient([[feat]], pts, calibs=cal, precision="fp32")
    auto = net.query_gradient([[feat]], pts, calibs=cal, precision="auto")
    assert torch.equal(auto[0], exact[0]) and torch.equal(auto[1], exact[1])
    with pytest.raises(RuntimeError, match="65536 texels"):
        net.query_gradient([[feat]], pts, calibs=cal, precision="tc")
