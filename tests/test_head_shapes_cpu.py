"""CPU tier of the head goldens (tests/golden/head_*.npz): heads other than the two shipped ones -- tiles of 32, 16 and 8
points, the two exactly full tiles and the next width up, widths that are not multiples of 4 or 32, fewer than 32 features,
one layer and eight, outputs other than 1 and 3, no last op, no skip inputs -- through the exact kernels of query_fp32.cu
compiled unmodified on the CPU model of tests/emu (the query, the point gradient and the surface render), against the
reference and the restatement.  And the tensor-core program's default feature limit per last op, on the shipped widths."""
import subprocess

import pytest
import torch

from oracle import spec
from grad_cases import query_grad_ref, within_bar
from emu_harness import build, run
from head_cases import (fp32_tile, head_cases, head_grad_cases, head_widths, load_head_case, load_head_grad_case,
                        shipped_widths)

TC_PAIRS = [(net, op) for net in ("G", "C") for op in (spec.LAST_SIGMOID, spec.LAST_TANH, spec.LAST_NONE)]


def _widths(chans, no_residual=False):
    return ("noskip:" if no_residual else "") + ",".join(str(c) for c in chans[1:])


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return dict(fp32=build(tmp_path_factory, "emu_fp32"), tc=build(tmp_path_factory, "emu_tc"))


def _launch(exe, tmp_path, c, n, op, shape, sms=3, extra=(), widths=None, points=None, returncode=0):
    """-> (out, the finished process) of emu_fp32 with the head's widths"""
    inp = dict(feat=c["feat"], rows=c["points"][:, :, :n] if points is None else points, calib=c["calib"], proj=c["proj"],
               res=c["chans"][-1], last_op=c["last_op"], Ws=c["Ws"], bs=c["bs"])
    return run(exe, tmp_path, op, *extra, inp=inp, shape=shape, options=dict(widths=widths or _widths(c["chans"]), sms=sms),
               returncode=returncode)


def _tiles(stdout):
    return [int(line.split("=")[1]) for line in stdout.split() if line.startswith("P=")]


def _query(exe, tmp_path, c, n, sms=3):
    out, r = _launch(exe, tmp_path, c, n, "query", (c["chans"][-1], n), sms)
    return out, _tiles(r.stdout)


def _grad(exe, tmp_path, c, n, sms=3):
    res = c["chans"][-1]
    out, r = _launch(exe, tmp_path, c, n, "grad", ((res + 3) * n,), sms)
    return out[:res * n].reshape(res, n), out[res * n:].reshape(3, n), _tiles(r.stdout)


def _fp32_heads():
    """the goldens of heads the tensor-core programs do not run (the others are the last-op pairs of the shipped widths)"""
    return [n for n in head_cases() if shipped_widths(head_widths(n)) is None]


# ---- the goldens and the restatement -----------------------------------------------------------------------------------
def test_head_goldens_cover_the_edges():
    cs = {n: load_head_case(n) for n in head_cases()}
    chans = {n: c["chans"] for n, c in cs.items()}
    tiles = {n: fp32_tile(ch) for n, ch in chans.items() if cs[n]["net"] is None}
    assert set(tiles.values()) == {32, 16, 8}
    assert any(ch[0] - 1 < 32 and (ch[0] - 1) % 32 for ch in chans.values()), "a map of fewer than 32 channels, not 32k"
    assert any(any(w % 32 for w in ch[1:-1]) for ch in chans.values()), "a hidden width that is not a multiple of 32"
    assert any(any(w % 4 for w in ch[1:-1]) for ch in chans.values()), "a hidden width that is not a multiple of 4"
    assert {len(ch) - 1 for ch in chans.values()} >= {1, 8}, "one layer and MP_MAX_LAYERS"
    assert any(ch[-1] not in (1, 3) for ch in chans.values())
    assert {(c["net"], c["last_op"]) for c in cs.values() if c["net"]} == set(TC_PAIRS) - {("G", spec.LAST_SIGMOID),
                                                                                         ("C", spec.LAST_TANH)}
    assert any(c["last_op"] == spec.LAST_NONE for c in cs.values() if c["net"] is None)
    assert fp32_tile(chans["p32_full"]) == 32 and fp32_tile(chans["p32_full"][:2] + [chans["p32_full"][2] + 1] + [1]) == 16
    assert fp32_tile(chans["p8_full"]) == 8 and fp32_tile([1025, 4096, 2072, 1]) is None
    assert fp32_tile(chans["p8_full"], grad=True) is None
    assert set(head_grad_cases()) == {n for n in tiles if fp32_tile(chans[n], grad=True)}


@pytest.mark.parametrize("name", head_cases())
def test_restatement_matches_head_golden(name):
    c = load_head_case(name)
    want = spec.query_ref(c["feat"], c["points"], c["calib"], c["Ws"], c["bs"], c["last_op"], c["proj"])
    assert (want - c["expected"]).abs().max().item() < 2e-6
    if c["amax"] is not None:
        assert c["feat"].abs().max().item() == pytest.approx(c["amax"], rel=1e-6)


@pytest.mark.parametrize("name", head_grad_cases())
def test_grad_restatement_matches_head_golden(name):
    c = load_head_grad_case(name)
    _, g64 = query_grad_ref(c["feat"], c["points"], c["calib"], c["Ws"], c["bs"], c["last_op"], c["proj"], dtype=torch.float64)
    assert (g64 - c["grad64"]).abs().max().item() <= 1e-9 * c["grad64"].abs().max().item()
    val, _ = query_grad_ref(c["feat"], c["points"], c["calib"], c["Ws"], c["bs"], c["last_op"], c["proj"])
    assert (val - c["value"]).abs().max().item() < 2e-6


# ---- the exact kernels on the CPU model ----------------------------------------------------------------------------------
def _n(c):
    return c["points"].shape[2]


@pytest.mark.parametrize("name", _fp32_heads())
def test_fp32_kernel_matches_head_golden(emu, tmp_path, name):
    """within 2e-5 * max(1, max|ref|) of the reference, out-of-image points exactly 0, and the tile the footprint predicts"""
    c = load_head_case(name)
    got, tiles = _query(emu["fp32"], tmp_path, c, _n(c))
    want = c["expected"]
    err = (got - want).abs().max().item()
    assert err <= 2e-5 * max(1.0, want.abs().max().item()), err
    zero = want == 0
    assert bool(zero.any()) and torch.equal(got[zero], want[zero]), "out-of-image points must be exactly 0"
    assert tiles == [fp32_tile(c["chans"])]


@pytest.mark.parametrize("name", head_grad_cases())
def test_grad_kernel_matches_head_golden(emu, tmp_path, name):
    """the point gradient within its bar of the reference's fp32 autograd, its value the query's bit for bit, and the
    gradient's tile the footprint predicts (the masks and g make it smaller than the query's for p32_full)"""
    c = load_head_grad_case(name)
    n = _n(c)
    val, dp, tiles = _grad(emu["fp32"], tmp_path, c, n)
    assert (val - c["value"]).abs().max().item() <= 2e-5 * max(1.0, c["value"].abs().max().item())
    ok, msg = within_bar(dp, c["grad32"])
    assert ok, msg
    ok, msg = within_bar(dp, c["grad64"])
    assert ok, "against fp64: " + msg
    q, _ = _query(emu["fp32"], tmp_path, c, n)
    assert torch.equal(val, q)
    assert tiles == [fp32_tile(c["chans"]), fp32_tile(c["chans"], grad=True)]


@pytest.mark.parametrize("name", ["narrow", "odd", "single"])
def test_results_do_not_depend_on_the_sm_count(emu, tmp_path, name):
    """1, 2 and 3 simulated SMs (one CTA walks all 17 tiles, or they interleave): the same bits, query and gradient"""
    c = load_head_grad_case(name)
    n = _n(c)
    q = [_query(emu["fp32"], tmp_path, c, n, sms)[0] for sms in (1, 2, 3)]
    g = [_grad(emu["fp32"], tmp_path, c, n, sms)[1] for sms in (1, 2, 3)]
    assert torch.equal(q[0], q[1]) and torch.equal(q[0], q[2])
    assert torch.equal(g[0], g[1]) and torch.equal(g[0], g[2])


R_CANVAS = 33


@pytest.mark.parametrize("name", ["single", "g_res3"])
def test_surface_render_of_a_three_output_head(emu, tmp_path, name):
    """The exact surface render with a 3-output head of one layer and with the geometry widths' 3-output head (Tanh): 90
    vertices of a 33^3 box against the restatement of colorization() driven by the oracle's query."""
    c = load_head_case(name)
    g = torch.Generator().manual_seed(11)
    n = 90
    cols = torch.randperm(R_CANVAS * R_CANVAS, generator=g)[:n]
    X, Y = cols // R_CANVAS, cols % R_CANVAS
    Z = torch.rand(n, generator=g) * (R_CANVAS - 1)
    rows = torch.stack([X.float(), Y.float(), Z])[None]
    got, _ = _launch(emu["fp32"], tmp_path, c, n, "surface", (R_CANVAS, R_CANVAS, 3), 2, [R_CANVAS, n, -1, -1, -1, 1, 1, 1],
                     points=rows)

    def query_c(points, calib):
        return spec.query_ref(c["feat"], points, calib, c["Ws"], c["bs"], c["last_op"], c["proj"])

    want = spec.colorization_ref(query_c, X, Y, Z, c["calib"], resolution=R_CANVAS)
    assert (got - want).abs().max().item() <= 2e-5
    untouched = torch.ones(R_CANVAS, R_CANVAS, dtype=torch.bool)
    untouched[X, Y] = False
    assert bool((got[untouched] == 1.0).all())


# ---- refusals ------------------------------------------------------------------------------------------------------------
def _zero_head(chans, last_op=spec.LAST_SIGMOID):
    """a head of these widths with zero weights, on a 2 x 3 map, 8 points (for the launchers' refusals)"""
    Ws = [torch.zeros(chans[l + 1], chans[l] + (chans[0] if l else 0)) for l in range(len(chans) - 1)]
    bs = [torch.zeros(chans[l + 1]) for l in range(len(chans) - 1)]
    return dict(chans=chans, last_op=last_op, Ws=Ws, bs=bs, feat=torch.zeros(1, chans[0] - 1, 2, 3),
                points=torch.zeros(1, 3, 8), calib=None, proj="orthogonal")


@pytest.mark.parametrize("chans,mode,what", [
    ([1025, 4096, 2072, 1], "query", "fp32 kernel"),          # one past the exactly full P = 8 tile
    ([9, 8192, 1], "query", "fp32 kernel"),
    ([1025, 4096, 2071, 1], "grad", "gradient kernel"),       # p8_full: its query runs, its gradient does not fit
])
def test_one_past_each_fit_is_refused(emu, tmp_path, chans, mode, what):
    _, r = _launch(emu["fp32"], tmp_path, _zero_head(chans), 8, mode, None, returncode=3)
    assert r.returncode == 3 and "head too wide for the %s's shared-memory tiling (-3)" % what in r.stderr, r.stderr


@pytest.mark.parametrize("mode", ["query", "grad"])
def test_no_residual_head_is_refused(emu, tmp_path, mode):
    c = load_head_case("narrow")
    nr = dict(c, Ws=[torch.zeros(c["chans"][l + 1], c["chans"][l]) for l in range(3)])
    _, r = _launch(emu["fp32"], tmp_path, nr, 8, mode, None, widths=_widths(c["chans"], no_residual=True), returncode=3)
    assert r.returncode == 3 and "no_residual heads are not supported (-3)" in r.stderr, r.stderr


# ---- the tensor-core program's default feature limit, per last op -------------------------------------------------------
def _default_limit(exe, res, last_op):
    r = subprocess.run([exe, "limit", str(res), str(last_op)], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stderr
    return float(r.stdout)


def test_shipped_pairs_keep_their_limits(emu):
    assert _default_limit(emu["fp32"], 1, spec.LAST_SIGMOID) == 12.0
    assert _default_limit(emu["fp32"], 3, spec.LAST_TANH) == 8.0


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("net,last_op", [p for p in TC_PAIRS if p != ("C", spec.LAST_TANH)])
def test_tc_program_within_the_bar_at_the_default_limit(emu, tmp_path, net, last_op, seed):
    """Each last op on the shipped widths, a seeded 32 x 32 map scaled to 0.99 x the head's default feature limit (what
    `auto` still sends to the tensor cores), 512 points on 2 simulated SMs: within 1e-4 of the fp32 oracle.  (A small map
    is the harder case: scaled to the same max |feature|, its features are larger on average than a 128 x 128 map's.)
    The colour head's Tanh keeps its shipped limit of 8, which reaches 1.2e-4 here (DESIGN.md §F1, range guard)."""
    chans = spec.G_CHANNELS if net == "G" else spec.C_CHANNELS
    limit = _default_limit(emu["fp32"], chans[-1], last_op)
    Ws, bs = spec.make_weights(chans, 1000 + seed)
    feat = spec.make_feat(chans[0] - 1, 32, 32, 2000 + seed)
    feat = feat * (0.99 * limit / feat.abs().max().item())
    pts = spec.make_points(512, 3000 + seed)
    cal = spec.scene_calib(20, -60 + 17 * seed)
    inp = dict(feat=feat, rows=pts, calib=cal, proj="orthogonal", res=chans[-1], last_op=last_op, Ws=Ws, bs=bs)
    got, _ = run(emu["tc"], tmp_path, "query", inp=inp, shape=(chans[-1], 512), options=dict(sms=2))
    err = (got - spec.query_ref(feat, pts, cal, Ws, bs, last_op)).abs().max().item()
    assert err <= 1e-4, (limit, err)
