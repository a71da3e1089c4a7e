"""GPU tests of MonoPortNet.query_stages' backward off the goldens' shapes: the ordered feature gradient where an image of a
batch and the same image alone take different radix-pass counts (3 against 2, and 4 against 3 with keys of 2^24 and more),
per-layer partial weight / bias requests through the C-ABI, hidden units whose pre-activation is exactly 0, the input
layouts query_stages takes, and query_gradient's point gradient against query_stages' on every head gradient golden."""
import ctypes

import pytest
import torch

from head_cases import build_head_net, head_grad_cases, load_head_grad_case
from ordered_cases import GPU_RADIX_CASES, NARROW, radix_passes_rule, spread_case, zero_unit_case
from vjp_cases import build_vjp_net, flat, query_vjp_ref, rel_dist, vjp_bar

pytestmark = pytest.mark.gpu


@pytest.fixture
def deterministic():
    """torch's deterministic mode for the test, then whatever it was before"""
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)


def _net(c):
    return build_vjp_net(c["chans"], c["last_op"], c["Ws"], c["bs"], c["proj"])


def _run(net, c, want=("f", "p", "w")):
    """query_stages on stage 0 of a case, backward of sum(gout * pred) -> (pred, dfeat, dpoints, [dW_l], [db_l])"""
    f = c["feats"][0].cuda().requires_grad_("f" in want)
    p = c["points"].cuda().requires_grad_("p" in want)
    cal = None if c["calib"] is None else c["calib"].cuda()
    head = net.surface_classifier
    for t in head.parameters():
        t.requires_grad_("w" in want)
        t.grad = None
    pred = net.query_stages([[f]], p, cal)[0]
    (pred * c["grad_output"][0].cuda()).sum().backward()
    for t in head.parameters():
        t.requires_grad_(True)
    return (pred.detach(), f.grad, p.grad, [None if x.weight.grad is None else x.weight.grad[:, :, 0] for x in head.filters],
            [x.bias.grad for x in head.filters])


def _ref(c, dtype):
    return query_vjp_ref(c["feats"], c["points"], c["calib"], c["Ws"], c["bs"], c["last_op"], c["proj"], c["grad_output"],
                         dtype=dtype)


# ---- radix-pass counts -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(GPU_RADIX_CASES))
def test_an_image_of_a_batch_is_that_image_alone_at_another_pass_count(deterministic, name):
    """one chunk: image b's columns keep their relative order, so its ordered sums are the same bits in the batch and
    alone, though the batch's keys take one more radix pass"""
    B, H, W, N, bands = GPU_RADIX_CASES[name]
    assert radix_passes_rule(B * H * W) == radix_passes_rule(H * W) + 1
    c = spread_case(B, N, H, W, bands=bands, seed=len(name))
    net = _net(c)
    net.vjp_chunk_points = 1 << 30
    batch = _run(net, c, want=("f",))[1]
    assert batch.abs().max().item() > 0
    for b in range(B):
        cb = dict(c, feats=[c["feats"][0][b:b + 1]], points=c["points"][b:b + 1], grad_output=[c["grad_output"][0][b:b + 1]])
        alone = _run(net, cb, want=("f",))[1]
        assert torch.equal(batch[b:b + 1], alone), b
    if radix_passes_rule(B * H * W) < 4:
        return
    # the last image's points: keys of 2^24 and more (its rows from 2191 on), keys below, outside points and a crowded cell
    u, v = c["points"][B - 1, 0].double(), c["points"][B - 1, 1].double()
    inside = (u.abs() <= 1) & (v.abs() <= 1)
    row = ((v + 1) * 0.5 * (H - 1)).floor()
    key = (B - 1) * H * W + row * W + ((u + 1) * 0.5 * (W - 1)).floor()
    assert bool((inside & (key >= 1 << 24)).any()) and bool((inside & (key < 1 << 24) & (row >= 2100)).any())
    assert bool((~inside).any())
    runs = [batch] + [_run(net, c, want=("f",))[1] for _ in range(4)]
    for r in runs[1:]:
        assert torch.equal(r, runs[0])
    r64, r32 = _ref(c, torch.float64), _ref(c, torch.float32)
    ok, msg = vjp_bar(batch.cpu(), r64["dfeat"][0], rel_dist(r32["dfeat"][0], r64["dfeat"][0]))
    assert ok, msg


# ---- per-layer partial requests through the C-ABI --------------------------------------------------------------------------
FULL = 0b11111
# (d W mask, d b mask) over the 5 layers of the odd head: null d W for some layers, null d b for others, one layer entirely
# null, the first, the last, and a single layer's d W with another's d b
PARTIAL = [(0b10101, FULL), (FULL, 0b01010), (FULL & ~0b00100, FULL & ~0b00100), (FULL & ~1, FULL & ~1),
           (FULL & ~0b10000, FULL & ~0b10000), (0b00010, 0b01000)]


@pytest.mark.parametrize("flags", [0, 1])
def test_partial_requests_through_the_c_abi(flags):
    """mp_query_points_vjp_ex with null d W / d b entries: every array passed is the full request's bits, every other one
    keeps its sentinel"""
    from monoport_b200 import _lib
    from monoport_b200.modeling.MonoPortNet import FeatureHandle
    c = spread_case(2, 300, 11, 6, chans=[20, 300, 77, 130, 5, 2], seed=21)
    net = _net(c)
    lib = _lib.load()
    mlp = net.surface_classifier.handle()
    feat = c["feats"][0].cuda()
    B, C, H, W = feat.shape
    fh = FeatureHandle(C, H, W, feat.device, B=B)
    fh.upload(feat)
    pts = c["points"].cuda().contiguous()
    gout = c["grad_output"][0].cuda().contiguous()
    n = pts.shape[2]
    nbytes = lib.mp_query_points_vjp_scratch_bytes_ex(mlp, fh.ptr, B, n, 64, 1, 1, flags)
    assert nbytes > 0
    scratch = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    shapes = [tuple(w.shape) for w in c["Ws"]]

    def call(wm, bm):
        dfeat = torch.full((B, C, H, W), -7.0, device="cuda")
        dp = torch.full((B, 3, n), -7.0, device="cuda")
        dws = [torch.full(s, -7.0, device="cuda") for s in shapes]
        dbs = [torch.full(s[:1], -7.0, device="cuda") for s in shapes]
        wp = (ctypes.c_void_p * 5)(*[t.data_ptr() if (wm >> l) & 1 else None for l, t in enumerate(dws)])
        bp = (ctypes.c_void_p * 5)(*[t.data_ptr() if (bm >> l) & 1 else None for l, t in enumerate(dbs)])
        _lib.check(lib.mp_query_points_vjp_ex(
            mlp, fh.ptr, B, ctypes.c_void_p(pts.data_ptr()), n, 3 * n, n, 1, None, _lib.PROJ_ORTHOGONAL,
            ctypes.c_float(net.normalizer.scale), ctypes.c_void_p(gout.data_ptr()), ctypes.c_void_p(dfeat.data_ptr()),
            ctypes.c_void_p(dp.data_ptr()), wp, bp, ctypes.c_void_p(scratch.data_ptr()), nbytes, flags,
            _lib.stream_ptr(feat.device)), "mp_query_points_vjp_ex")
        torch.cuda.synchronize()
        return dfeat, dp, dws, dbs

    full = call(FULL, FULL)
    assert all(bool((t != 0).any()) and not bool((t == -7.0).any()) for t in full[2] + full[3])
    r64 = _ref(c, torch.float64)
    for g, got in (("dW", full[2]), ("db", full[3])):
        ok, msg = vjp_bar([t.cpu() for t in got], r64[g])
        assert ok, (g, msg)
    for wm, bm in PARTIAL:
        got = call(wm, bm)
        assert torch.equal(got[1], full[1])
        if flags:
            assert torch.equal(got[0], full[0])
        else:
            assert (got[0] - full[0]).abs().max().item() <= 1e-6 * full[0].abs().max().item()
        for l in range(5):
            for mask, x, y in ((wm, got[2][l], full[2][l]), (bm, got[3][l], full[3][l])):
                if (mask >> l) & 1:
                    assert torch.equal(x, y), (wm, bm, l)
                else:
                    assert bool((x == -7.0).all()), (wm, bm, l)
    del fh


# ---- pre-activations of exactly 0 ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("det", [False, True])
def test_pre_activations_of_exactly_zero_take_the_slope_at_zero(det):
    """lrelu' at 0 is the negative slope, as in torch's autograd: query_stages' gradients and query_gradient's point
    gradient within their bars of the float64 restatement, the zero units' rows within the bar of their own scale"""
    c, zero_rows = zero_unit_case()
    net = _net(c)
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        _, dfeat, dp, dW, db = _run(net, c)
    finally:
        torch.use_deterministic_algorithms(was)
    r64, r32 = _ref(c, torch.float64), _ref(c, torch.float32)
    for g, got in (("dfeat", [dfeat]), ("dpoints", dp), ("dW", dW), ("db", db)):
        ok, msg = vjp_bar(flat(got), r64[g], rel_dist(r32[g], r64[g]))
        assert ok, (g, msg)
    for l, rows in zero_rows.items():
        for g, got in (("dW", dW), ("db", db)):
            ref = r64[g][l][rows]
            assert ref.abs().max().item() > 0
            ok, msg = vjp_bar(got[l][rows].cpu(), ref, rel_dist(r32[g][l][rows], ref))
            assert ok, (l, g, msg)
    z0 = c["points"][:, 2] == 0
    ref = r64["dpoints"][:, 2][z0]
    ok, msg = vjp_bar(dp.cpu()[:, 2][z0], ref, rel_dist(r32["dpoints"][:, 2][z0], ref))
    assert ok, msg
    # query_gradient in fp32 (grad_output = ones), one image
    c1 = dict(c, feats=[c["feats"][0][:1]], points=c["points"][:1], grad_output=None)
    net.eval().precision = "fp32"
    _, g = net.query_gradient([[c1["feats"][0].cuda()]], c1["points"].cuda(), precision="fp32")
    q64, q32 = _ref(c1, torch.float64), _ref(c1, torch.float32)
    ok, msg = vjp_bar(g.cpu(), q64["dpoints"], rel_dist(q32["dpoints"], q64["dpoints"]))
    assert ok, msg
    z0 = c1["points"][:, 2] == 0
    ok, msg = vjp_bar(g.cpu()[:, 2][z0], q64["dpoints"][:, 2][z0],
                      rel_dist(q32["dpoints"][:, 2][z0], q64["dpoints"][:, 2][z0]))
    assert ok, msg


# ---- input layouts ---------------------------------------------------------------------------------------------------------
LAYOUTS = ["channels_last", "float64", "bfloat16", "transposed_points", "mean_loss"]


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_input_layouts_give_the_contiguous_float32_gradients(layout, det):
    """against the contiguous float32 run on the same values: the values, d points, d W and d b the same bits; d features
    the same bits in deterministic mode, within 1e-6 * max of them with atomics (and, in bfloat16, the rounding of either);
    every gradient in its input's dtype and shape"""
    c = spread_case(2, 500, 24, 20, chans=NARROW, seed=31)
    # values every dtype holds exactly
    feat = c["feats"][0].bfloat16().float().cuda()
    pts = c["points"].bfloat16().float().cuda()
    net = _net(c)
    gout = c["grad_output"][0].cuda()
    if layout == "mean_loss":
        gout = torch.full_like(gout, 1.0 / gout.numel())

    def run(f, p_leaf, p_arg, loss):
        head = net.surface_classifier
        for t in head.parameters():
            t.grad = None
        pred = net.query_stages([[f]], p_arg(p_leaf), None)[0]
        loss(pred).backward()
        return (pred.detach(), f.grad, p_leaf.grad, [x.weight.grad for x in head.filters], [x.bias.grad for x in head.filters])

    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        weighted = (lambda pred: (pred * gout).sum())
        base = run(feat.clone().requires_grad_(), pts.clone().requires_grad_(), lambda p: p, weighted)
        dtype = {"float64": torch.float64, "bfloat16": torch.bfloat16}.get(layout, torch.float32)
        f = feat.to(dtype)
        if layout == "channels_last":
            f = f.contiguous(memory_format=torch.channels_last)
            assert not f.is_contiguous()
        f.requires_grad_()
        if layout == "transposed_points":
            p_leaf, p_arg = pts.transpose(1, 2).contiguous().requires_grad_(), (lambda p: p.transpose(1, 2))
        else:
            p_leaf, p_arg = pts.to(dtype).requires_grad_(), (lambda p: p)
        got = run(f, p_leaf, p_arg, (lambda pred: pred.mean()) if layout == "mean_loss" else weighted)
    finally:
        torch.use_deterministic_algorithms(was)
    assert torch.equal(got[0], base[0])
    assert got[1].dtype == f.dtype and got[1].shape == f.shape
    assert got[2].dtype == p_leaf.dtype and got[2].shape == p_leaf.shape
    want_dp = base[2].transpose(1, 2) if layout == "transposed_points" else base[2]
    assert torch.equal(got[2], want_dp.to(got[2].dtype))
    for x, y in zip(got[3] + got[4], base[3] + base[4]):
        assert x.dtype == torch.float32 and torch.equal(x, y)
    want_df = base[1].to(got[1].dtype)
    if det:
        assert torch.equal(got[1], want_df)
    else:
        tol = 1e-6 * base[1].abs().max().item()
        if layout == "bfloat16":
            tol = tol + 2.0 ** -8 * base[1].abs()
        assert bool(((got[1].float() - want_df.float()).abs() <= tol).all())


# ---- the point gradient of query_gradient and query_stages -----------------------------------------------------------------
@pytest.mark.parametrize("name", head_grad_cases())
def test_query_gradient_is_query_stages_point_gradient_bit_for_bit(name):
    """every head gradient golden, reverse tile 8 included: the same kernel, the same bits"""
    c = load_head_grad_case(name)
    net = build_head_net(c)
    feat, pts = c["feat"].cuda(), c["points"].cuda()
    cal = c["calib"].cuda() if c["calib"] is not None else None
    _, want = net.query_gradient([[feat]], pts, calibs=cal, precision="fp32")
    p = pts.clone().requires_grad_()
    pred = net.query_stages([[feat]], p, cal)[0]
    pred.backward(torch.ones_like(pred))
    assert torch.equal(p.grad, want)
