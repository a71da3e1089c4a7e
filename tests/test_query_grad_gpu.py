"""GPU tests of the point gradient of query() (MonoPortNet.query_gradient -> mp_query_points_grad): the reference's autograd
goldens, the value against query() in fp32 mode bit for bit, the call's argument handling, and the two places that use it --
reconstruction(normals=True) and surface_normals() -- on the synthetic person."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import spec
from helpers import build_net
from grad_cases import grad_cases, load_grad_case, within_bar

pytestmark = pytest.mark.gpu


def _case_inputs(c):
    net = build_net(c)
    gout = c["grad_output"][None].cuda() if c["grad_output"] is not None else None
    cal = c["calib"].cuda() if c["calib"] is not None else None
    return net, [[c["feat"].cuda()]], c["points"].cuda(), cal, gout


@pytest.mark.parametrize("name", grad_cases())
def test_query_gradient_matches_reference_grad_golden(name):
    c = load_grad_case(name)
    net, feats, pts, cal, gout = _case_inputs(c)
    val, dp = net.query_gradient(feats, pts, calibs=cal, grad_output=gout)
    assert val.shape == (1, c["chans"][-1], pts.shape[2]) and dp.shape == (1, 3, pts.shape[2])
    assert (val[0].cpu() - c["value"]).abs().max().item() <= 2e-5
    ok, msg = within_bar(dp[0].cpu(), c["grad32"])
    assert ok, msg
    # exactly zero outside the image
    outside = (c["value"] == 0).all(0)
    assert bool((dp[0].cpu()[:, outside] == 0).all())


@pytest.mark.parametrize("name", ["g_rot", "g_persp", "c_rot"])
def test_value_is_query_fp32_bit_for_bit(name):
    c = load_grad_case(name)
    net, feats, pts, cal, gout = _case_inputs(c)
    net.precision = "fp32"
    want = net.query(feats, pts, calibs=cal)[0]
    val, _ = net.query_gradient(feats, pts, calibs=cal, grad_output=gout)
    assert torch.equal(val, want)


def test_grad_output_none_equals_ones():
    c = load_grad_case("g_rot")
    net, feats, pts, cal, _ = _case_inputs(c)
    a = net.query_gradient(feats, pts, calibs=cal)
    b = net.query_gradient(feats, pts, calibs=cal, grad_output=torch.ones(1, 1, pts.shape[2], device="cuda"))
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_strided_points_empty_input_and_argument_checks():
    c = load_grad_case("c_rot")
    net, feats, pts, cal, gout = _case_inputs(c)
    want = net.query_gradient(feats, pts, calibs=cal, grad_output=gout)
    view = pts[0].t().contiguous().t()[None]                 # the [N,3] layout RTL/main.py:176-177 passes, as a [1,3,N] view
    assert view.stride(2) == 3
    got = net.query_gradient(feats, view, calibs=cal, grad_output=gout)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    v0, d0 = net.query_gradient(feats, pts[:, :, :0], calibs=cal)
    assert v0.shape == (1, 3, 0) and d0.shape == (1, 3, 0)
    with pytest.raises(ValueError):
        net.query_gradient(feats, pts[0], calibs=cal)
    with pytest.raises(ValueError):
        net.query_gradient(feats, pts, calibs=cal, grad_output=gout[:, :1])
    with pytest.raises(NotImplementedError):
        net.train().query_gradient(feats, pts, calibs=cal)
    net.eval()
    with pytest.raises(RuntimeError):
        net.query_gradient([[c["feat"]]], pts, calibs=cal)


def test_batch_handle_is_refused():
    from monoport_b200 import _lib
    c = load_grad_case("g_nocalib")
    net = build_net(c)
    feat = torch.cat([c["feat"], c["feat"]], 0).cuda()
    fh = net.batch_feature_handle(feat)
    pts = c["points"][0].cuda().contiguous()
    dp = torch.empty(3, pts.shape[1], device="cuda")
    lib = _lib.load()
    rc = lib.mp_query_points_grad(net.surface_classifier.handle(), fh.ptr, ctypes.c_void_p(pts.data_ptr()), pts.shape[1],
                                  pts.shape[1], 1, None, 0, ctypes.c_float(spec.Z_SCALE), None, 0, None, 0,
                                  ctypes.c_void_p(dp.data_ptr()), pts.shape[1], _lib.stream_ptr())
    assert rc == -1 and b"single-map" in lib.mp_last_error()
    with pytest.raises(ValueError):
        net.query_gradient([[feat]], pts[None])


# ---- normals on the synthetic person (spec.heightfield_person) at R = 65 ------------------------------------------------
@pytest.fixture(scope="module")
def person():
    Ws, bs = spec.make_weights(spec.G_CHANNELS, 3)
    feat = spec.make_feat(256, 128, 128, 4, 0.5)
    Ws, bs, feat, _ = spec.heightfield_person(Ws, bs, feat)
    net = build_net("G", Ws, bs)
    net.precision = "fp32"
    return net, [[feat.cuda()]], spec.scene_calib(20, 0).cuda()


def test_reconstruction_normals(person):
    from monoport_b200.recon import reconstruction
    net, feats, cal = person
    R = 65
    lo, hi = [-1, -1, -1], [1, 1, 1]
    plain = reconstruction(net, "cuda:0", cal, R, lo, hi, feats=feats)
    assert plain != -1 and plain[2] is None and plain[3] is None
    verts, faces, nrm, vals = reconstruction(net, "cuda:0", cal, R, lo, hi, feats=feats, normals=True)
    assert torch.equal(verts, plain[0]) and torch.equal(faces, plain[1]) and vals is None
    assert nrm.shape == verts.shape and nrm.dtype == torch.float32
    length = nrm.norm(dim=1)
    nonzero = length > 0
    assert nonzero.double().mean().item() >= 0.99
    assert (length[nonzero] - 1).abs().max().item() <= 1e-5
    # outward: sigma falls through 0.5 along +n over half a voxel each way
    eps = 0.5 * 2.0 / R
    sig = lambda p: net.query(feats, p.t().unsqueeze(0).contiguous(), calibs=cal)[0][0, 0]
    out_ = sig(verts + eps * nrm)
    in_ = sig(verts - eps * nrm)
    frac = ((out_ < 0.5) & (in_ > 0.5)).double().mean().item()
    print("sign test: %.4f of %d vertices" % (frac, verts.shape[0]))
    assert frac >= 0.99
    # against central differences of the fp32 field, h = 1e-3
    h = 1e-3
    fd = torch.stack([sig(verts + h * e) - sig(verts - h * e) for e in torch.eye(3, device="cuda")], 1) / (2 * h)
    fdn = -fd / fd.norm(dim=1, keepdim=True)
    cos = (fdn * nrm).sum(1)
    q = torch.quantile(cos[torch.isfinite(cos)], torch.tensor([0.01, 0.1, 0.5], device="cuda")).tolist()
    print("cosine with central differences: 1%% %.5f  10%% %.5f  median %.6f" % tuple(q))
    assert q[2] >= 0.999
    # normals follow a rigid transform like the vertices do
    T = torch.eye(4)
    T[:3, :3] = torch.from_numpy(spec._rot(0.3, -0.7, 0.2)).float()
    T[:3, 3] = torch.tensor([0.5, -1.0, 2.0])
    tv, _, tn, _ = reconstruction(net, "cuda:0", cal, R, lo, hi, feats=feats, normals=True, transform=T)
    Tc = T.cuda()
    assert torch.allclose(tv, verts @ Tc[:3, :3].T + Tc[:3, 3], atol=1e-5)
    assert torch.allclose(tn, nrm @ Tc[:3, :3].T, atol=1e-5)


def test_surface_normals_agree_with_forward_vertices(person):
    from monoport_b200.recon import colorization, forward_vertices, surface_normals
    net, feats, cal = person
    R = 65
    vol = net.query_grid(feats[-1][0], cal, R, torch.tensor([-1.0] * 3), torch.tensor([1.0] * 3))
    X, Y, Z, fvn = forward_vertices(vol[None, None], "front")
    assert X.numel() > 100
    nrm = surface_normals(net, feats, X, Y, Z, cal, resolution=R)
    assert nrm.shape == fvn.shape
    ok = torch.isfinite(fvn).all(1) & (nrm.norm(dim=1) > 0)
    cos = (nrm[ok] * fvn[ok]).sum(1)
    print("surface_normals vs forward_vertices: mean cosine %.4f, median %.4f over %d vertices"
          % (cos.mean().item(), cos.median().item(), int(ok.sum())))
    assert cos.mean().item() >= 0.9
    img = colorization(None, None, X, Y, Z, cal, norm=nrm, resolution=R)
    assert img.shape == (R, R, 3)
    assert torch.allclose(img[X, Y, :], ((nrm + 1) / 2).clamp(0, 1))
    assert surface_normals(net, feats, None, None, None, cal) is None
