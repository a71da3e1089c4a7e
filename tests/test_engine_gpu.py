"""GPU parity of the coarse-to-fine engines (csrc/octree.cu), marching cubes and the visible-surface kernel against
the oracle restatements (bit-exact indices / topology) and the reference goldens (forward_vertices)."""
import glob
import os

import numpy as np
import pytest
import torch

from oracle import spec
from helpers import GOLDEN, build_net, lookup_query

pytestmark = pytest.mark.gpu

RES = [9, 17, 33, 65]
UNIT = ((-1.0, -1.0, -1.0), (1.0, 1.0, 1.0))
B1 = ((-0.83, -1.17, -0.61), (0.91, 1.06, 0.77))          # asymmetric, no power-of-two extent
B_PIFU = ((-128.0, -28.0, -128.0), (128.0, 228.0, 128.0))  # upstream PIFu's reconstruction box


def _engine(kind, fn, box=UNIT, balance=0.5, **kw):
    from monoport_b200.engine import Seg3dLossless, Seg3dTopk
    b_min = np.array([box[0]], dtype=np.float32)
    b_max = np.array([box[1]], dtype=np.float32)
    if kind == "topk":
        return Seg3dTopk(query_func=fn, b_min=b_min, b_max=b_max, resolutions=RES, balance_value=balance, **kw).to("cuda")
    return Seg3dLossless(query_func=fn, b_min=b_min, b_max=b_max, resolutions=RES, balance_value=balance,
                         use_cuda_impl=False, faster=(kind == "faster")).to("cuda")


@pytest.mark.parametrize("field_kind,box,balance", [
    pytest.param("sphere", UNIT, 0.5, id="sphere"), pytest.param("two_blobs", UNIT, 0.5, id="two_blobs"),
    pytest.param("ellipsoid", UNIT, 0.5, id="ellipsoid"),
    # boxes whose three extents differ (a swapped or shared axis extent changes the points), other balances, fields that
    # reach the box and nodes equal to the balance
    pytest.param("sphere", B1, 0.5, id="sphere-B1"), pytest.param("corner", B1, 0.3, id="corner-B1-0.3"),
    pytest.param("slab", B1, 0.7, id="slab-B1-0.7"), pytest.param("steps", B1, 0.3, id="steps-B1-0.3"),
    pytest.param("noise", B1, 0.7, id="noise-B1-0.7"), pytest.param("steps", B_PIFU, 0.5, id="steps-PIFU"),
    pytest.param("noise", B_PIFU, 0.3, id="noise-PIFU-0.3"), pytest.param("corner", B_PIFU, 0.7, id="corner-PIFU-0.7"),
    pytest.param("slab", B_PIFU, 0.5, id="slab-PIFU")])
@pytest.mark.parametrize("kind", ["faster", "lossless", "topk"])
def test_engine_matches_oracle_bit_exact(kind, field_kind, box, balance):
    field = torch.from_numpy(spec.analytic_volume(65, field_kind))
    fn_o, fn_e = lookup_query(field, *box)
    recorded = []

    def fn_rec(points, **kw):
        recorded.append(points[0].clone())
        return fn_e(points)

    if kind == "topk":
        kpts = [0, 2500, 9000, 40000]
        want, stats = spec.seg3d_topk_ref(fn_o, RES, kpts, *box, balance=balance, return_stats=True)
        eng = _engine("topk", fn_rec, box, balance, num_points=kpts)
    else:
        want, stats = spec.seg3d_lossless_ref(fn_o, RES, *box, balance=balance, faster=(kind == "faster"), return_stats=True)
        eng = _engine(kind, fn_rec, box, balance)
    got = eng(anything="goes")                        # unknown kwargs are forwarded (RTL/main.py:392-394)
    assert got.shape == (1, 1, 65, 65, 65) and got.device.type == "cuda"
    assert torch.equal(got[0, 0].cpu(), want), "volume must be bit-identical to the restatement"
    # per-level node counts and the exact world points handed to query_func (== index sets, in order)
    assert eng.last_stats == [int(s["idx"].numel()) for s in stats]
    got_pts = torch.cat(recorded).cpu()
    want_pts = []
    for s in stats:
        res, idx = s["res"], s["idx"]
        if idx.numel() == 0:
            continue
        stride = 64 // (res - 1)
        c = torch.stack([idx % res, (idx // res) % res, idx // (res * res)], 1) * stride
        want_pts.append(spec.level_points(c, 65, *box))
    assert torch.equal(got_pts, torch.cat(want_pts)), "evaluated node sets / order differ"


def test_engine_returns_none_on_empty_volume():
    fn_o, fn_e = lookup_query(torch.zeros(65, 65, 65))
    for kind in ("faster", "lossless"):
        assert _engine(kind, fn_e)() is None
    assert _engine("topk", fn_e, num_points=[0, 10, 10, 10])() is None


def test_lossless_property_at_full_size():
    """257^3, lossless mode: the octree mask must equal the dense mask while evaluating a small fraction of nodes."""
    from monoport_b200.engine import Seg3dLossless
    field = torch.from_numpy(spec.analytic_volume(257, "two_blobs"))
    fn_o, fn_e = lookup_query(field)
    b = np.array([[-1.0, -1.0, -1.0]], dtype=np.float32)
    eng = Seg3dLossless(fn_e, b, -b, [17, 33, 65, 129, 257], balance_value=0.5, faster=False).to("cuda")
    got = eng()
    assert torch.equal((got[0, 0] > 0.5).cpu(), field > 0.5)
    assert sum(eng.last_stats) < 0.05 * 257 ** 3
    eng_f = Seg3dLossless(fn_e, b, -b, [17, 33, 65, 129, 257], balance_value=0.5, faster=True).to("cuda")
    gf = eng_f()
    assert eng_f.last_stats[-1] == 0
    assert ((gf[0, 0] > 0.5).cpu() != (field > 0.5)).float().mean().item() < 1e-3


def test_fused_engine_equals_generic_engine_with_mlp():
    """The fused on-device pyramid and the generic Python-callback pyramid must give the same volume when the
    callback is the net itself (fp32 mode => bit-identical)."""
    from monoport_b200.engine import Seg3dLossless, make_query_func
    Ws, bs = spec.make_weights(spec.G_CHANNELS, 3)
    feat = spec.make_feat(256, 128, 128, 4, 0.5)
    Ws, bs, feat, _ = spec.heightfield_person(Ws, bs, feat)
    net = build_net("G", Ws, bs)
    cal = spec.scene_calib(20, 33).cuda()
    feats = [[feat.cuda()]]
    b = np.array([[-1.0, -1.0, -1.0]], dtype=np.float32)
    res = [17, 33, 65, 129]
    for mode in (["fp32", "tc", "tc_v3"] if net.surface_classifier.tc_supported() else ["fp32"]):
        net.precision = mode
        for faster in (True, False):
            fused = Seg3dLossless(make_query_func(net), b, -b, res, balance_value=0.5, faster=faster).to("cuda")

            def plain(points, im_feat_list, calib_tensor):          # RTL/main.py:168-183 without the fused tag
                return net.query(im_feat_list, points=points.permute(0, 2, 1), calibs=calib_tensor)[0]

            generic = Seg3dLossless(plain, b, -b, res, balance_value=0.5, faster=faster).to("cuda")
            a = fused(im_feat_list=feats, calib_tensor=cal)
            g = generic(im_feat_list=feats, calib_tensor=cal)
            assert a is not None and g is not None
            assert fused.last_stats == generic.last_stats, (mode, faster, fused.last_stats, generic.last_stats)
            assert torch.equal(a, g), (mode, faster)
            if mode == "fp32" and not faster:
                # against the oracle engine driven by the oracle query (CPU, fp32): same mask
                def q(p):
                    return spec.query_ref(feat, p.t().contiguous(), cal.cpu(), Ws, bs, spec.LAST_SIGMOID)[0]
                want = spec.seg3d_lossless_ref(q, res, faster=False)
                assert ((a[0, 0].cpu() > 0.5) != (want > 0.5)).sum().item() <= 2   # fp32 summation-order ties only


@pytest.mark.parametrize("kind,R,iso", [
    pytest.param("sphere", 33, 0.5, id="sphere-33"), pytest.param("two_blobs", 65, 0.5, id="two_blobs-65"),
    pytest.param("ellipsoid", 40, 0.5, id="ellipsoid-40"),
    # nodes equal to the iso value; surfaces cut by the volume's faces; dense noise on odd and tiny shapes
    pytest.param("steps", 33, 0.5, id="steps-33"), pytest.param("steps", 33, 0.25, id="steps-33-iso0.25"),
    pytest.param("corner", 65, 0.5, id="corner-65"), pytest.param("noise", (20, 17, 23), 0.5, id="noise-20x17x23"),
    pytest.param("noise", (3, 70, 2), 0.5, id="noise-3x70x2"), pytest.param("noise", (2, 3, 257), 0.5, id="noise-2x3x257"),
    pytest.param("noise", (9, 40, 35), 0.5, id="noise-9x40x35")])
def test_marching_cubes_matches_oracle(kind, R, iso):
    from monoport_b200.recon import marching_cubes
    if kind == "noise":          # (the shapes of the CPU model's noise cases, same generator)
        vol = np.random.default_rng(sum(R)).random(R, dtype=np.float32)
    else:
        vol = spec.analytic_volume(R, kind)
    V, F = spec.marching_cubes_ref(vol, iso)
    v, f = marching_cubes(torch.from_numpy(vol).cuda(), iso)
    assert len(F) > 0
    assert f.dtype == torch.int32 and np.array_equal(f.cpu().numpy(), F), "topology must be bit-exact"
    assert np.abs(v.cpu().numpy() - V).max() <= 1e-6


def test_marching_cubes_full_size_watertight():
    from monoport_b200.recon import marching_cubes
    vol = torch.from_numpy(spec.analytic_volume(257, "two_blobs")).cuda()
    v, f = marching_cubes(vol)
    f = f.long()
    assert f.min() >= 0 and f.max() == v.shape[0] - 1
    e = torch.cat([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    key = e[:, 0] * v.shape[0] + e[:, 1]
    rkey = e[:, 1] * v.shape[0] + e[:, 0]
    assert key.unique().numel() == key.numel()                    # every directed edge once ...
    assert torch.equal(key.sort().values, rkey.sort().values)     # ... and its reverse once => closed + oriented
    und = torch.minimum(key, rkey).unique().numel()
    assert v.shape[0] - und + f.shape[0] == 4                     # two spheres
    a, b, c = v[f[:, 0]].double(), v[f[:, 1]].double(), v[f[:, 2]].double()
    assert ((a * torch.cross(b, c, dim=1)).sum() > 0)
    assert marching_cubes(torch.zeros(9, 9, 9, device="cuda"))[0].shape[0] == 0


@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(GOLDEN, "fv_*.npz"))))
def test_forward_vertices_matches_reference_golden(path):
    from monoport_b200.recon import forward_vertices
    g = np.load(path)
    vol = torch.from_numpy(spec.analytic_volume(int(g["R"]), str(g["kind"])))[None, None].cuda()
    for d in ("front", "back", "left", "right"):
        X, Y, Z, n = forward_vertices(vol, d)
        assert X.dtype == torch.int64 and np.array_equal(X.cpu().numpy(), g["X_" + d])
        assert np.array_equal(Y.cpu().numpy(), g["Y_" + d])
        np.testing.assert_allclose(Z.cpu().numpy(), g["Z_" + d], rtol=0, atol=1e-5, equal_nan=True)
        np.testing.assert_allclose(n.cpu().numpy(), g["N_" + d], rtol=0, atol=1e-6, equal_nan=True)
    assert forward_vertices(None) == (None, None, None, None)


def test_forward_vertices_full_size_vs_oracle():
    from monoport_b200.recon import forward_vertices
    vol = torch.from_numpy(spec.analytic_volume(257, "ellipsoid"))[None, None]
    for d in ("front", "right"):
        X, Y, Z, n = forward_vertices(vol.cuda(), d)
        Xo, Yo, Zo, no = spec.forward_vertices_ref(vol, d)
        assert torch.equal(X.cpu(), Xo) and torch.equal(Y.cpu(), Yo)
        assert torch.allclose(Z.cpu(), Zo, atol=1e-4, equal_nan=True)
        assert torch.allclose(n.cpu(), no, atol=1e-6, equal_nan=True)


def test_reconstruction_dense_vs_octree():
    from monoport_b200.recon import reconstruction
    Ws, bs = spec.make_weights(spec.G_CHANNELS, 3)
    feat = spec.make_feat(256, 128, 128, 4, 0.5)
    Ws, bs, feat, _ = spec.heightfield_person(Ws, bs, feat)
    net = build_net("G", Ws, bs)
    net.precision = "fp32"
    cal = spec.scene_calib(20, 0).cuda()
    feats = [[feat.cuda()]]
    dense = reconstruction(net, "cuda:0", cal, 65, [-1, -1, -1], [1, 1, 1], feats=feats)
    octree = reconstruction(net, "cuda:0", cal, 65, [-1, -1, -1], [1, 1, 1], use_octree=True, feats=feats)
    assert dense != -1 and octree != -1
    assert torch.equal(dense[1], octree[1]) and torch.allclose(dense[0], octree[0], atol=1e-5)
    assert dense[0].abs().max() <= 1.0


def test_colorization_matches_restatement():
    """netC colour pass of the demo (RTL/main.py:212-249): visible vertices -> world -> netC.query -> canvas."""
    from monoport_b200.recon import forward_vertices, colorization
    Wc, bc = spec.make_weights(spec.C_CHANNELS, 21)
    featc = spec.make_feat(512, 128, 128, 22)
    netC = build_net("C", Wc, bc)
    vol = torch.from_numpy(spec.analytic_volume(65, "ellipsoid"))[None, None]
    cal = spec.scene_calib(20, 33)
    X, Y, Z, n = forward_vertices(vol.cuda(), "front")
    img = colorization(netC, [[featc.cuda()]], X, Y, Z, cal.cuda(), resolution=65)

    def qc(points, calib):
        return spec.query_ref(featc, points, calib, Wc, bc, spec.LAST_TANH)
    Xo, Yo, Zo, _ = spec.forward_vertices_ref(vol, "front")
    want = spec.colorization_ref(qc, Xo, Yo, Zo, cal, resolution=65)
    assert img.shape == (65, 65, 3)
    assert (img.cpu() - want).abs().max().item() <= 5e-5
    imgn = colorization(netC, None, X, Y, Z, cal.cuda(), norm=n, resolution=65)
    wantn = spec.colorization_ref(None, Xo, Yo, Zo, cal, resolution=65, norm=spec.forward_vertices_ref(vol, "front")[3])
    assert torch.allclose(imgn.cpu(), wantn, atol=1e-6, equal_nan=True)
    assert colorization(netC, None, None, None, None, cal.cuda()) is None


def test_frame_pipeline_overlap_equals_sequential():
    """processors=[...] pipeline with 2 overlapping lanes (threads + streams) == the same stages run sequentially."""
    from monoport_b200.engine import Seg3dLossless, make_query_func
    from monoport_b200.pipeline import FramePipeline
    from monoport_b200.recon import forward_vertices
    Ws, bs = spec.make_weights(spec.G_CHANNELS, 3)
    base = spec.make_feat(256, 128, 128, 4, 0.5)
    feats = []
    for k in range(3):
        W2, b2, f, _ = spec.heightfield_person(Ws, bs, base * (1.0 + 0.1 * k), channel=0)
        feats.append(f.cuda())
    net = build_net("G", W2, b2)
    net.precision = "tc"
    cal = spec.scene_calib(20, 33).cuda()
    b = np.array([[-1.0, -1.0, -1.0]], dtype=np.float32)
    eng = Seg3dLossless(make_query_func(net), b, -b, [17, 33, 65], balance_value=0.5, faster=True).to("cuda")

    def recon_stage(f):
        return eng(im_feat_list=[[f]], calib_tensor=cal)

    def surf_stage(sdf):
        X, Y, Z, n = forward_vertices(sdf, "front")
        return sdf, X, Y, Z

    seq = [surf_stage(recon_stage(f)) for f in (feats * 3)]
    pipe = FramePipeline([recon_stage, surf_stage], "cuda:0", n_lanes=2)
    par = list(pipe.run(f for f in (feats * 3)))
    pipe.close()
    assert len(par) == len(seq) == 9
    for a, c in zip(seq, par):
        assert torch.equal(a[0], c[0]) and torch.equal(a[1], c[1]) and torch.equal(a[3], c[3])


def test_frame_graph_equals_eager_frames():
    """SURVEY.md 8f-2: the CUDA-graph captured frame step (features -> coarse-to-fine engine -> visible surface, one graph
    launch per frame, two lanes in flight) returns exactly what the eager calls return, frame after frame, including an
    empty frame (engine -> None) between full ones; and with the PyTorch encoder inside the captured step."""
    from monoport_b200.engine import Seg3dLossless, make_query_func
    from monoport_b200.pipeline import FrameGraph, FrameGraphRing
    from monoport_b200.recon import forward_vertices
    Ws, bs = spec.make_weights(spec.G_CHANNELS, 3)
    base = spec.make_feat(256, 128, 128, 4, 0.5)
    feats = []
    for k in range(3):
        W2, b2, f, _ = spec.heightfield_person(Ws, bs, base * (1.0 + 0.1 * k), channel=0)
        feats.append(f.cuda())
    empty = feats[0].clone()
    empty[0, 0] = -5.0                                   # height map far below every node: nothing occupied
    frames = [feats[0], feats[1], empty, feats[2], feats[0]]
    net = build_net("G", W2, b2)
    cal = spec.scene_calib(20, 33)
    b = np.array([[-1.0, -1.0, -1.0]], dtype=np.float32)
    eng = Seg3dLossless(make_query_func(net), b, -b, [17, 33, 65], balance_value=0.5, faster=True).to("cuda")
    want = []
    for f in frames:
        sdf = eng(im_feat_list=[[f]], calib_tensor=cal.cuda())
        X, Y, Z, n = forward_vertices(sdf, "front")
        want.append((None if sdf is None else sdf.clone(), X, Y, Z, n, list(eng.last_stats)))
    assert want[2][0] is None and want[0][0] is not None
    ring = FrameGraphRing(lambda: FrameGraph(net, eng, cal, "front", with_encoder=False), n_lanes=2)
    got = []
    for sdf, X, Y, Z, n in ring.run(iter(frames)):
        got.append((None if sdf is None else sdf.clone(), None if X is None else X.clone(), None if Z is None else Z.clone(),
                    None if n is None else n.clone()))
    assert len(got) == len(want)
    for w, g in zip(want, got):
        if w[0] is None:
            assert g[0] is None
            continue
        assert torch.equal(w[0], g[0]) and torch.equal(w[1], g[1]) and torch.equal(w[3], g[2]) and torch.equal(w[4], g[3])
    assert ring.lanes[0].last_stats == want[4][5]
    ring.close()
    # with the encoder inside the captured step: same volume as filter() + engine() run eagerly on the same image
    torch.manual_seed(0)
    net.image_filter.cuda()
    img = (torch.rand(1, 3, 512, 512, generator=torch.Generator().manual_seed(5)) * 2 - 1).cuda()

    def hook(f):                                          # deterministic body-like field: channel 0 carries the height map
        f = f.clone()
        f[:, 0] = feats[0][:, 0]
        return f
    with torch.no_grad():
        fe = hook(net.filter(img)[-1][0])
        sdf = eng(im_feat_list=[[fe]], calib_tensor=cal.cuda())
    fg = FrameGraph(net, eng, cal, "front", with_encoder=True, feature_hook=hook)
    for _ in range(2):
        out = fg.launch(img).result()
        assert out[0] is not None and sdf is not None
        # cudnn may pick another algorithm under capture: the encoder output agrees to float noise, the mask to a few nodes
        assert ((out[0] > 0.5) != (sdf > 0.5)).sum().item() <= 64
    fg.close()
