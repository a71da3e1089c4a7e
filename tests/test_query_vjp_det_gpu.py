"""GPU tests of the ordered feature gradient of MonoPortNet.query_stages under torch.use_deterministic_algorithms(True): the
reference's goldens, the same bits from run to run and for every request, the other gradients the bits of the atomic
path, an image of a batch against the same image alone, and 20 000 points in one cell against the float64 restatement."""
import pytest
import torch

from oracle import spec
from ordered_cases import one_cell_case
from vjp_cases import build_vjp_net, flat, golden_bar, load_vjp_case, query_vjp_ref, rel_dist, vjp_bar, vjp_cases

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


def _run(net, c, want=("f", "p", "w")):
    """query_stages over every stage of a case, backward of sum(gout * preds) -> (dfeat [S], dpoints, dW [L], db [L]); the
    gradients not in `want` are not requested (None)"""
    fs = [f.cuda().requires_grad_("f" in want) for f in c["feats"]]
    p = c["points"].cuda().requires_grad_("p" in want)
    cal = None if c["calib"] is None else c["calib"].cuda()
    head = net.surface_classifier
    for t in head.parameters():
        t.requires_grad_("w" in want)
        t.grad = None
    preds = net.query_stages([[f] for f in fs], p, cal)
    gout = c["grad_output"]
    total = sum((pr * (torch.ones_like(pr) if gout is None else gout[s].cuda())).sum() for s, pr in enumerate(preds))
    total.backward()
    for t in head.parameters():
        t.requires_grad_(True)
    return ([f.grad for f in fs], p.grad, [None if f.weight.grad is None else f.weight.grad[:, :, 0] for f in head.filters],
            [f.bias.grad for f in head.filters])


def _net(c):
    return build_vjp_net(c["chans"], c["last_op"], c["Ws"], c["bs"], c["proj"])


@pytest.mark.parametrize("name", vjp_cases())
def test_ordered_gradients_match_reference_vjp_golden(deterministic, name):
    c = load_vjp_case(name)
    dfeat, dp, dW, db = _run(_net(c), c)
    for g, got in (("dfeat", dfeat), ("dpoints", dp), ("dW", dW), ("db", db)):
        ok, msg = golden_bar(flat(got), c, g)
        assert ok, msg


def test_five_runs_and_every_request_give_the_same_bits(deterministic):
    c = load_vjp_case("g_b3_s4_persp")
    net = _net(c)
    net.vjp_chunk_points = 96                      # several chunks per stage
    runs = [_run(net, c) for _ in range(5)]
    for r in runs[1:]:
        for x, y in zip(r[0], runs[0][0]):
            assert torch.equal(x, y)
        assert torch.equal(r[1], runs[0][1])
        for x, y in zip(r[2] + r[3], runs[0][2] + runs[0][3]):
            assert torch.equal(x, y)
    only_f = _run(net, c, want=("f",))
    assert only_f[1] is None
    for x, y in zip(only_f[0], runs[0][0]):
        assert torch.equal(x, y)
    # the other three gradients are the bits of the atomic path; d features its sums up to their order
    torch.use_deterministic_algorithms(False)
    off = _run(net, c)
    torch.use_deterministic_algorithms(True)
    assert torch.equal(off[1], runs[0][1])
    for x, y in zip(off[2] + off[3], runs[0][2] + runs[0][3]):
        assert torch.equal(x, y)
    for x, y in zip(off[0], runs[0][0]):
        assert (x - y).abs().max().item() <= 1e-6 * x.abs().max().item()


@pytest.mark.parametrize("kind", ["G", "C"])
def test_an_image_of_a_batch_is_that_image_alone(deterministic, kind):
    """one chunk: image b of a B = 3 batch and the same image, points and calib as a batch of one"""
    c = load_vjp_case("g_b3_s4_persp" if kind == "G" else "c_b3_rot")
    c = dict(c, feats=c["feats"][:1], grad_output=None if c["grad_output"] is None else c["grad_output"][:1])
    net = _net(c)
    net.vjp_chunk_points = 1 << 30
    batch = _run(net, c, want=("f",))[0][0]
    for b in range(3):
        cb = dict(c, feats=[c["feats"][0][b:b + 1]], points=c["points"][b:b + 1],
                  calib=None if c["calib"] is None else c["calib"][b:b + 1],
                  grad_output=None if c["grad_output"] is None else [c["grad_output"][0][b:b + 1]])
        alone = _run(net, cb, want=("f",))[0][0]
        assert torch.equal(batch[b:b + 1], alone), b


def test_twenty_thousand_points_in_one_cell(deterministic):
    c = one_cell_case(1, 20000, 32, 32, chans=spec.G_CHANNELS, seed=1)
    net = _net(c)
    runs = [_run(net, c, want=("f",))[0][0] for _ in range(2)]
    assert torch.equal(runs[0], runs[1])
    args = (c["feats"], c["points"], c["calib"], c["Ws"], c["bs"], c["last_op"], c["proj"], c["grad_output"])
    r64, r32 = query_vjp_ref(*args, dtype=torch.float64), query_vjp_ref(*args, dtype=torch.float32)
    ok, msg = vjp_bar(runs[0], r64["dfeat"][0], rel_dist(r32["dfeat"][0], r64["dfeat"][0]))
    assert ok, msg
