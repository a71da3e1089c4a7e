"""The demo's display images (visulization, RTL/main.py:252-281) inside the captured frame: FrameGraph(display=True) ends its
step with mp_display_async on the lane's canvases, and displayed() returns page-locked numpy views.  recon.visulization,
the eager twin, equals the torch restatement on the GPU bit for bit; every ring frame's displayed() equals visulization of
the eager chain's images, for the three engines and each image configuration, over the AUTO cameras, an empty frame and a
colour frame on the exact route; and display=True leaves result(), rendered() and mesh() as they were."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import spec
from display_cases import visulization_ref
from helpers import build_net

pytestmark = pytest.mark.gpu

RES = [17, 33, 65]
AUTO = [spec.scene_calib(20, 3 * k) for k in range(6)]
B0, B1 = (-1.0, -1.0, -1.0), (1.0, 1.0, 1.0)


def _same_np(a, b):
    """numpy outputs: float32 bit for bit (NaN included), bool equal; None only against None"""
    if a is None or b is None:
        return a is None and b is None
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype == np.float32:
        return np.array_equal(np.ascontiguousarray(a).view(np.int32), np.ascontiguousarray(b).view(np.int32))
    return np.array_equal(a, b)


def _same(a, b):
    if a is None or b is None:
        return a is None and b is None
    return a.shape == b.shape and bool(((a == b) | (torch.isnan(a) & torch.isnan(b))).all())


def _canvas(R, seed, bg=1.0):
    g = torch.Generator().manual_seed(seed)
    c = torch.full((R, R, 3), bg)
    fg = torch.rand(R, R, generator=g) < 0.5
    c[fg] = torch.randint(0, 17, (int(fg.sum()), 3), generator=g).float() / 16.0
    c[torch.rand(R, R, generator=g) < 0.01, 1] = float("nan")
    return c.cuda()


@pytest.mark.parametrize("R", [17, 65, 128, 129, 256, 257, 300, 513])
def test_visulization_equals_restatement(R):
    """recon.visulization = display_cases.visulization_ref run with torch on the GPU, bit for bit, for both images and each
    alone, with the reference's types and shapes."""
    from monoport_b200.recon import visulization
    norm, tex = _canvas(R, R), _canvas(R, R + 1, bg=0.5 if R % 2 else 1.0)
    for n, t in ((norm, tex), (norm, None), (None, tex)):
        got, want = visulization(n, t), visulization_ref(n, t)
        for a, b in zip(got, want):
            assert _same_np(a, b), R
        for img in got[:2]:
            assert img is None or (img.dtype == np.float32 and img.shape == (256, 256, 3))
        assert got[2].dtype == np.bool_ and got[2].shape == (256, 256, 1)
    assert visulization(None, None) == (None, None, None)
    assert visulization(norm)[1] is None


def _person():
    Ws, bs = spec.make_weights(spec.G_CHANNELS, 3)
    base = spec.make_feat(256, 128, 128, 4, 0.5)
    feats = []
    for k in range(2):
        W2, b2, f, _ = spec.heightfield_person(Ws, bs, base * (1.0 + 0.1 * k), channel=0)
        feats.append(f.cuda())
    return build_net("G", W2, b2), feats


def _engine(net, kind, res=RES):
    from monoport_b200.engine import Seg3dLossless, Seg3dTopk, make_query_func
    b = np.array([[-1.0, -1.0, -1.0]], dtype=np.float32)
    if kind == "topk":
        return Seg3dTopk(make_query_func(net), b, -b, RES, [0, 9000, 30000]).to("cuda")
    return Seg3dLossless(make_query_func(net), b, -b, res, balance_value=0.5, faster=kind == "faster").to("cuda")


def _out_of_image(cal):
    c = cal.clone()
    c[0, 0, 3] += 10.0
    return c


def test_visulization_of_the_test_persons_colorization():
    """On the eager colorization() images of the test person (normals and netC colours): bit for bit the restatement."""
    from monoport_b200.recon import colorization, forward_vertices, visulization
    net, feats = _person()
    netC = build_net("C", *spec.make_weights(spec.C_CHANNELS, 21))
    eng = _engine(net, "faster")
    cal = AUTO[1].cuda()
    sdf = eng(im_feat_list=[[feats[0]]], calib_tensor=cal)
    X, Y, Z, N = forward_vertices(sdf, "front")
    rnorm = colorization(netC, None, X, Y, Z, cal, norm=N, resolution=RES[-1])
    rtex = colorization(netC, [[spec.make_feat(512, 128, 128, 22, 0.5).cuda()]], X, Y, Z, cal, resolution=RES[-1])
    for n, t in ((rnorm, rtex), (rnorm, None), (None, rtex)):
        got = visulization(n, t)
        assert got[2].any() and not got[2].all()
        for a, b in zip(got, visulization_ref(n, t)):
            assert _same_np(a, b)


IMAGES = {"netC+normals": dict(netC=True, render_normals=True), "netC+gradient": dict(netC=True, render_normals="gradient"),
          "normals": dict(netC=False, render_normals=True), "netC": dict(netC=True, render_normals=False)}


def _eager_images(net, netC, eng, f, c, cal, render_normals, R):
    """the eager chain's (render_norm, render_tex) of one frame, or None for an empty frame"""
    from monoport_b200.recon import colorization, forward_vertices, surface_normals
    sdf = eng(im_feat_list=[[f]], calib_tensor=cal)
    if sdf is None:
        return None
    X, Y, Z, N = forward_vertices(sdf.clone(), "front")
    rnorm = None
    if render_normals:
        Nn = N if render_normals is True else surface_normals(net, [[f]], X, Y, Z, cal, R, B0, B1, precision="auto")
        rnorm = colorization(None, None, X, Y, Z, cal, norm=Nn, resolution=R)
    rtex = colorization(netC, [[c]], X, Y, Z, cal, resolution=R) if netC is not None else None
    return rnorm, rtex


def _run_ring(kind, lanes, images, res=RES, mesh=False, n_frames=None):
    from monoport_b200.pipeline import FrameGraph, FrameGraphRing
    from monoport_b200.recon import visulization
    net, feats = _person()
    cfg = IMAGES[images]
    netC = build_net("C", *spec.make_weights(spec.C_CHANNELS, 21)) if cfg["netC"] else None
    eng = _engine(net, kind, res)
    R = res[-1]
    c0 = spec.make_feat(512, 128, 128, 22, 0.5).cuda()
    big = c0 * 60.0                                       # far above the colour head's limit: the exact route
    cams = AUTO[:3] + [_out_of_image(AUTO[3])] + AUTO[4:]
    colours = [c0, c0, big, c0, c0, big]
    frames = list(zip([feats[k % 2] for k in range(len(cams))], colours))[:n_frames]
    cams = cams[:n_frames]
    want = [_eager_images(net, netC, eng, f, c, cal.cuda(), cfg["render_normals"], R) for (f, c), cal in zip(frames, cams)]
    assert sum(w is None for w in want) <= 1 and want[0] is not None

    def make(display):
        return lambda: FrameGraph(net, eng, AUTO[0], "front", with_encoder=False, netC=netC,
                                  render_normals=cfg["render_normals"], mesh=mesh, display=display)
    items = frames if netC is not None else [f for f, _ in frames]
    plain = FrameGraphRing(make(False), n_lanes=lanes)
    plain_out = [tuple(None if t is None else t.clone() for t in out) for out in plain.run(items, calibs=cams)]
    plain.close()
    ring = FrameGraphRing(make(True), n_lanes=lanes)
    n = 0
    for i, (w, p, out) in enumerate(zip(want, plain_out, ring.run(items, calibs=cams))):
        n += 1
        assert len(out) == len(p) + 3, (i, len(out), len(p))
        for k, (a, b) in enumerate(zip(p, out)):                          # result(), rendered(), mesh() unchanged
            assert _same(a, b), (kind, images, i, k)
        shown = out[len(p):]
        if w is None:
            assert shown == (None, None, None) and out[0] is None
            continue
        for k, (a, b) in enumerate(zip(out[5:7], w)):                     # rendered() is the eager chain's
            assert _same(a, b), (kind, images, i, k)
        for ref in (visulization(*w), visulization_ref(*w)):
            for k, (a, b) in enumerate(zip(shown, ref)):
                assert _same_np(a, b), (kind, images, i, k)
    assert n == len(frames)
    ring.close()


@pytest.mark.parametrize("kind,lanes,images", [
    ("faster", 1, "netC+normals"), ("faster", 2, "netC+normals"), ("faster", 2, "netC+gradient"), ("faster", 2, "normals"),
    ("faster", 1, "netC"), ("lossless", 1, "netC+gradient"), ("lossless", 2, "netC+normals"), ("lossless", 2, "normals"),
    ("topk", 1, "normals"), ("topk", 2, "netC+gradient"), ("topk", 2, "netC")])
def test_ring_displays_what_the_eager_chain_shows(kind, lanes, images):
    """Every frame over the AUTO cameras, an empty frame and colour frames on the exact route: displayed() =
    visulization(*the eager chain's images) bit for bit (NaN positions included), and the outputs before it are those of
    the same ring built without display."""
    _run_ring(kind, lanes, images)


def test_ring_with_mesh_and_display():
    """display=True next to mesh=True: mesh() is unchanged and displayed() follows the mesh outputs."""
    _run_ring("faster", 2, "netC+normals", mesh=True, n_frames=4)


def test_display_upscales_a_129_engine_on_the_device():
    """An engine that ends at 129^3: 129 -> 256 nearest upscale inside the captured step."""
    _run_ring("faster", 1, "netC+normals", res=[17, 33, 65, 129], n_frames=3)


def test_refusals():
    from monoport_b200 import _lib
    from monoport_b200.pipeline import FrameGraph
    net, feats = _person()
    eng = _engine(net, "faster")
    with pytest.raises(ValueError):
        FrameGraph(net, eng, AUTO[0], "front", with_encoder=False, display=True)
    g = FrameGraph(net, eng, AUTO[0], "front", with_encoder=False, render_normals=True, display=True)
    with pytest.raises(RuntimeError):
        g.displayed()                                     # before result()
    g.launch(feats[0]).result()
    assert g.displayed()[0] is not None and g.displayed()[1] is None
    g.close()
    plain = FrameGraph(net, eng, AUTO[0], "front", with_encoder=False, render_normals=True)
    plain.launch(feats[0]).result()
    with pytest.raises(RuntimeError):
        plain.displayed()                                 # a graph built without display
    plain.close()
    # the C ABI: pageable host outputs, both images NULL; page-locked outputs are accepted
    lib = _lib.load()
    R, S = 33, 256
    canvas = torch.ones((R, R, 3), device="cuda")
    staging = torch.empty(7 * S * S, device="cuda")
    st = _lib.stream_ptr()

    def p(t):
        return ctypes.c_void_p(t.data_ptr() if torch.is_tensor(t) else t.ctypes.data)
    pinned = [torch.empty(n, dtype=dt, pin_memory=True) for n, dt in ((3 * S * S, torch.float32), (3 * S * S, torch.float32),
                                                                      (S * S, torch.uint8))]
    pageable = [np.empty(3 * S * S, np.float32), np.empty(3 * S * S, np.float32), np.empty(S * S, np.uint8)]
    assert lib.mp_display_async(p(canvas), p(canvas), R, S, *map(p, pinned), p(staging), st) == _lib.MP_OK
    torch.cuda.synchronize()
    assert bool((pinned[0] == 255).all()) and not bool(pinned[2].any())
    for k in range(3):
        outs = list(map(p, pinned))
        outs[k] = p(pageable[k])
        assert lib.mp_display_async(p(canvas), p(canvas), R, S, *outs, p(staging), st) == -1, k
        assert b"page-locked" in lib.mp_last_error()
    assert lib.mp_display_async(None, None, R, S, *map(p, pinned), p(staging), st) == -1
    torch.cuda.synchronize()
