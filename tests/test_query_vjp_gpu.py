"""GPU tests of the differentiable query for training (MonoPortNet.query_stages -> mp_query_points_vjp): the reference's
autograd goldens, a float64 restatement of train-mode query() on small cases, values and point gradients bit for bit
against query() / query_gradient() in fp32, determinism of the weight / bias / point gradients, frozen parts, a short SGD loop
against the same loop on the fp32 restatement, and the refusals."""
import pytest
import torch
import torch.nn.functional as F

from oracle import spec
from helpers import build_net
from grad_cases import load_grad_case
from vjp_cases import (GRAD_NAMES, build_vjp_net, flat, golden_bar, load_vjp_case, query_vjp_ref, rel_dist, vjp_bar,
                       vjp_cases)

pytestmark = pytest.mark.gpu


def _run(net, feats, points, calib, gout=None):
    """query_stages on CUDA copies, backward of sum(gout * preds) -> (preds, dfeat [S], dpoints, dW [L], db [L])"""
    fs = [f.cuda().requires_grad_() for f in feats]
    p = points.cuda().requires_grad_()
    cal = None if calib is None else calib.cuda()
    preds = net.query_stages([[f] for f in fs], p, cal)
    total = sum((pr * (torch.ones_like(pr) if gout is None else gout[s].cuda())).sum() for s, pr in enumerate(preds))
    for f in net.surface_classifier.filters:
        f.weight.grad = None
        f.bias.grad = None
    total.backward()
    head = net.surface_classifier
    return ([pr.detach() for pr in preds], [f.grad for f in fs], p.grad, [f.weight.grad[:, :, 0] for f in head.filters],
            [f.bias.grad for f in head.filters])


def _small_case(chans, B, S, N, H, W, calib, last_op=spec.LAST_SIGMOID, seed=0, gout=True):
    Ws, bs = spec.make_weights(chans, 900 + seed)
    feats = [torch.cat([spec.make_feat(chans[0] - 1, H, W, 910 + seed + 10 * s + b) for b in range(B)]) for s in range(S)]
    points = torch.stack([spec.make_points(N, 920 + seed + b)[0] for b in range(B)])
    cal = None
    if calib != "none":
        cal = torch.stack([spec.scene_calib(15.0 + 10 * b, 25.0 - 5 * b)[0] for b in range(B)])
        if calib == "persp":
            cal[:, 2, 3] = 3.0
            cal[:, :2, :] *= 2.5
    g = None
    if gout:
        gen = torch.Generator().manual_seed(930 + seed)
        g = [torch.randn(B, chans[-1], N, generator=gen) for _ in range(S)]
    return dict(chans=chans, Ws=Ws, bs=bs, feats=feats, points=points, calib=cal, grad_output=g, last_op=last_op,
                proj="perspective" if calib == "persp" else "orthogonal")


SMALL = {
    "g_b1_rot": lambda: _small_case(spec.G_CHANNELS, 1, 1, 203, 32, 32, "rot", gout=False),
    "g_b3_s2_persp": lambda: _small_case(spec.G_CHANNELS, 3, 2, 97, 16, 24, "persp", seed=1),
    "c_b2_nocalib": lambda: _small_case(spec.C_CHANNELS, 2, 1, 70, 16, 16, "none", spec.LAST_TANH, seed=2),
    "narrow_none": lambda: _small_case([33, 48, 40, 2], 2, 2, 150, 20, 12, "rot", spec.LAST_NONE, seed=3),
}


@pytest.mark.parametrize("name", sorted(SMALL))
def test_matches_float64_restatement(name):
    c = SMALL[name]()
    net = build_vjp_net(c["chans"], c["last_op"], c["Ws"], c["bs"], c["proj"])
    preds, dfeat, dp, dW, db = _run(net, c["feats"], c["points"], c["calib"], c["grad_output"])
    args = (c["feats"], c["points"], c["calib"], c["Ws"], c["bs"], c["last_op"], c["proj"], c["grad_output"])
    r64 = query_vjp_ref(*args, dtype=torch.float64)
    r32 = query_vjp_ref(*args, dtype=torch.float32)
    for s, pr in enumerate(preds):
        assert (pr.cpu().double() - r64["value"][s]).abs().max().item() <= 2e-5
    for g, got in (("dfeat", dfeat), ("dpoints", dp), ("dW", dW), ("db", db)):
        ok, msg = vjp_bar(got, r64[g], rel_dist(r32[g], r64[g]))
        assert ok, (g, msg)


@pytest.mark.parametrize("name", vjp_cases())
def test_matches_reference_vjp_golden(name):
    c = load_vjp_case(name)
    net = build_vjp_net(c["chans"], c["last_op"], c["Ws"], c["bs"], c["proj"])
    preds, dfeat, dp, dW, db = _run(net, c["feats"], c["points"], c["calib"], c["grad_output"])
    assert (flat(preds) - c["value"].double().reshape(-1)).abs().max().item() <= 2e-5
    for g, got in (("dfeat", dfeat), ("dpoints", dp), ("dW", dW), ("db", db)):
        ok, msg = golden_bar(flat(got), c, g)
        assert ok, msg


@pytest.mark.parametrize("B", [1, 3])
def test_values_are_query_fp32_bit_for_bit(B):
    c = _small_case(spec.G_CHANNELS, B, 1, 300, 64, 64, "rot", seed=5)
    net = build_vjp_net(c["chans"], c["last_op"], c["Ws"], c["bs"])
    feat, pts, cal = c["feats"][0].cuda(), c["points"].cuda(), c["calib"].cuda()
    want = net.eval().query([[feat]], pts, cal)[0]
    got = net.train().query_stages([[feat.requires_grad_()]], pts, cal)[0]
    assert torch.equal(got.detach(), want)


@pytest.mark.parametrize("name", ["g_rot", "g_persp", "c_rot"])
def test_dpoints_are_query_gradient_bit_for_bit(name):
    c = load_grad_case(name)
    net = build_net(c)
    feat, pts = c["feat"].cuda(), c["points"].cuda()
    cal = c["calib"].cuda() if c["calib"] is not None else None
    gout = c["grad_output"][None].cuda() if c["grad_output"] is not None else None
    _, want = net.query_gradient([[feat]], pts, calibs=cal, grad_output=gout, precision="fp32")
    p = pts.clone().requires_grad_()
    pred = net.query_stages([[feat]], p, cal)[0]
    pred.backward(torch.ones_like(pred) if gout is None else gout)
    assert torch.equal(p.grad, want)


def test_weight_bias_point_gradients_are_deterministic_across_runs_and_chunks():
    c = _small_case(spec.G_CHANNELS, 2, 1, 1000, 32, 32, "rot", seed=6)
    net = build_vjp_net(c["chans"], c["last_op"], c["Ws"], c["bs"])
    one = _run(net, c["feats"], c["points"], c["calib"], c["grad_output"])
    net.vjp_chunk_points = 96                      # 21 chunks of the 2 x 1000 points
    a = _run(net, c["feats"], c["points"], c["calib"], c["grad_output"])
    b = _run(net, c["feats"], c["points"], c["calib"], c["grad_output"])
    assert torch.equal(a[2], b[2]) and torch.equal(a[2], one[2])          # d points: no contraction
    for x, y in zip(a[3] + a[4], b[3] + b[4]):
        assert torch.equal(x, y)
    ok, msg = vjp_bar(a[3], one[3])                  # another chunk size: another summation order
    assert ok, msg


def test_frozen_head_and_frozen_features_give_the_same_gradients():
    c = _small_case(spec.C_CHANNELS, 2, 1, 400, 32, 32, "rot", spec.LAST_TANH, seed=7)
    net = build_vjp_net(c["chans"], c["last_op"], c["Ws"], c["bs"])
    full = _run(net, c["feats"], c["points"], c["calib"], c["grad_output"])
    # frozen head: the same d points bit for bit, the same d features up to the atomics' order
    for p in net.surface_classifier.parameters():
        p.requires_grad_(False)
    fs = [f.cuda().requires_grad_() for f in c["feats"]]
    pts = c["points"].cuda().requires_grad_()
    pred = net.query_stages([[f] for f in fs], pts, c["calib"].cuda())[0]
    pred.backward(c["grad_output"][0].cuda())
    assert torch.equal(pts.grad, full[2])
    assert (fs[0].grad - full[1][0]).abs().max().item() <= 1e-6 * full[1][0].abs().max().item()
    for p in net.surface_classifier.parameters():
        p.requires_grad_(True)
    # frozen features and points: the same weight and bias gradients bit for bit
    pred = net.query_stages([[c["feats"][0].cuda()]], c["points"].cuda(), c["calib"].cuda())[0]
    head = net.surface_classifier
    gW = torch.autograd.grad(pred, [f.weight for f in head.filters] + [f.bias for f in head.filters],
                             grad_outputs=c["grad_output"][0].cuda())
    L = len(head.filters)
    for x, y in zip(gW[:L], full[3]):
        assert torch.equal(x[:, :, 0], y)
    for x, y in zip(gW[L:], full[4]):
        assert torch.equal(x, y)


@pytest.mark.parametrize("kind", ["G", "C"])
def test_sgd_loop_tracks_the_fp32_restatement(kind):
    chans = spec.G_CHANNELS if kind == "G" else spec.C_CHANNELS
    last_op = spec.LAST_SIGMOID if kind == "G" else spec.LAST_TANH
    c = _small_case(chans, 2, 1, 500, 32, 32, "rot", last_op, seed=8, gout=False)
    gen = torch.Generator().manual_seed(940)
    labels = torch.rand(2, chans[-1], 500, generator=gen) * (1.0 if kind == "G" else 2.0) - (0.0 if kind == "G" else 1.0)
    loss_fn = F.mse_loss if kind == "G" else F.l1_loss
    lr = 0.5 if kind == "G" else 0.05
    net = build_vjp_net(chans, last_op, c["Ws"], c["bs"])
    net.train()
    head = net.surface_classifier
    fmap = c["feats"][0].cuda().requires_grad_()
    opt = torch.optim.SGD(list(head.parameters()) + [fmap], lr=lr)
    # the same loop on the fp32 restatement
    Ws = [w.clone().cuda().requires_grad_() for w in c["Ws"]]
    bs = [b.clone().cuda().requires_grad_() for b in c["bs"]]
    fref = c["feats"][0].clone().cuda().requires_grad_()
    opt_ref = torch.optim.SGD(Ws + bs + [fref], lr=lr)
    pts, cal, lab = c["points"].cuda(), c["calib"].cuda(), labels.cuda()
    prev_tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        for step in range(5):
            opt.zero_grad()
            loss = loss_fn(net.query_stages([[fmap]], pts, cal)[0], lab)
            loss.backward()
            opt.step()
            opt_ref.zero_grad()
            outs = []
            for b in range(2):
                xyz = spec.project_ref(pts[b], cal[b])
                u, v, z = xyz[0], xyz[1], xyz[2]
                in_img = (u >= -1) & (u <= 1) & (v >= -1) & (v <= 1)
                x = torch.cat([spec.bilinear_ref(fref[b], u, v), (z * spec.Z_SCALE)[None]], 0)
                outs.append(in_img.float()[None] * spec.mlp_ref(x, Ws, bs, last_op))
            loss_ref = loss_fn(torch.stack(outs), lab)
            loss_ref.backward()
            opt_ref.step()
            assert abs(loss.item() - loss_ref.item()) <= 1e-5 * abs(loss_ref.item()) + 1e-7, (step, loss.item(), loss_ref.item())
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev_tf32
    for f, W, b in zip(head.filters, Ws, bs):
        assert (f.weight[:, :, 0] - W).abs().max().item() <= 1e-5 * W.abs().max().item()
        assert (f.bias - b).abs().max().item() <= 1e-5 * b.abs().max().item() + 1e-7
    assert (fmap - fref).abs().max().item() <= 1e-5 * fref.abs().max().item()


def test_refusals_and_unchanged_query():
    c = _small_case(spec.G_CHANNELS, 1, 1, 64, 16, 16, "rot", seed=9)
    net = build_vjp_net(c["chans"], c["last_op"], c["Ws"], c["bs"])
    feat = c["feats"][0].cuda().requires_grad_()
    pts, cal = c["points"].cuda(), c["calib"].cuda()
    with pytest.raises(ValueError):
        net.query_stages([[feat]], pts, cal.clone().requires_grad_())
    with pytest.raises(NotImplementedError):
        net.query_stages([[feat, feat]], pts, cal)
    with pytest.raises(NotImplementedError):
        net.query_stages([[feat]], pts, cal, transforms=torch.zeros(1, 2, 3, device="cuda"))
    with pytest.raises(NotImplementedError):
        net.train().query([[feat]], pts, cal)
    # no double backward
    pred = net.query_stages([[feat]], pts, cal)[0]
    (g,) = torch.autograd.grad(pred.sum(), feat, create_graph=True)
    with pytest.raises(RuntimeError):
        g.sum().backward()
    # an optimizer step between forward and backward: autograd's version error, not stale weights
    pred = net.query_stages([[feat]], pts, cal)[0]
    with torch.no_grad():
        net.surface_classifier.filters[0].weight.add_(1e-3)
    with pytest.raises(RuntimeError):
        pred.sum().backward()
    # the backward uploads the saved map again: another query in between changes nothing
    net.eval()
    feat2 = c["feats"][0].cuda().clone().requires_grad_()
    pred = net.query_stages([[feat2]], pts, cal)[0]
    pred.backward(torch.ones_like(pred))
    want = feat2.grad.clone()
    feat2.grad = None
    pred = net.query_stages([[feat2]], pts, cal)[0]
    net.query([[torch.randn_like(feat2)]], pts, cal)
    pred.backward(torch.ones_like(pred))
    assert (feat2.grad - want).abs().max().item() <= 1e-6 * want.abs().max().item()
