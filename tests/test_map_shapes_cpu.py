"""CPU tier of the map-shape goldens (tests/golden/shape_*.npz): feature maps that are not square (a swapped H and W shows),
whose texel count is not a multiple of 128 (the last, partial block of the per-texel G0 kernel), that have an axis of length 1,
or that sit at or above the tensor-core program's 65536 texels.  The restatement is pinned against the reference on all of
them, and the query kernels -- compiled unmodified on the CPU model of tests/emu -- against the reference and the restatement:
the tensor-core program with its per-texel products, the exact fp32 kernel, the point gradient and the colour surface render."""
import os

import numpy as np
import pytest
import torch

from oracle import spec
from emu_harness import build, run
from grad_cases import query_grad_ref, within_bar
from shape_cases import (TC_TEXEL_LIMIT, load_shape_batch_case, load_shape_case, load_shape_grad_case, shape_batch_cases,
                         shape_cases, shape_grad_cases, within_fp32_bar)
# one OS thread per CUDA thread is slow: the heaviest cases only run with MONOPORT_B200_EMU_FULL=1
FULL = os.environ.get("MONOPORT_B200_EMU_FULL", "0") == "1"
full_only = pytest.mark.skipif(not FULL, reason="heavy emulation case: set MONOPORT_B200_EMU_FULL=1")
N_CORNER = slice(8, 72)          # the points whose projections land on and next to the last row and column


# ---- the goldens and the restatement -----------------------------------------------------------------------------------
def test_shape_goldens_cover_the_shapes():
    """The properties the goldens exist for: H != W both ways, texel counts that are not a multiple of 128, an axis of
    length 1 both ways, maps of exactly 65536 texels (square and not) and maps above that, for both heads."""
    shapes = {n: (load_shape_case(n)["H"], load_shape_case(n)["W"], load_shape_case(n)["net"]) for n in shape_cases()}
    hw = {n: h * w for n, (h, w, _) in shapes.items()}
    assert any(h < w for h, w, _ in shapes.values()) and any(h > w for h, w, _ in shapes.values())
    assert any(h == 1 for h, _, _ in shapes.values()) and any(w == 1 for _, w, _ in shapes.values())
    assert {(h, w) for n, (h, w, _) in shapes.items() if hw[n] == TC_TEXEL_LIMIT} >= {(256, 256), (128, 512)}
    assert {net for n, (_, _, net) in shapes.items() if hw[n] > TC_TEXEL_LIMIT} == {"G", "C"}
    assert {net for n, (h, w, net) in shapes.items() if hw[n] % 128 and h != w and h > 1 and w > 1} == {"G", "C"}
    assert any(load_shape_case(n)["calib"] is None and h != w for n, (h, w, _) in shapes.items())
    assert set(shape_grad_cases()) >= {"g_wide", "g_tiny"} and shape_batch_cases()


@pytest.mark.parametrize("name", shape_cases())
def test_corner_cluster_reaches_the_last_texel_block(name):
    """The points right after the 8 border points sample the last texels in row-major order -- the last, partial block of
    128 texels when H * W % 128 != 0 --, the very last texel included: a G0 block that is not computed cannot hide."""
    c = load_shape_case(name)
    H, W = c["H"], c["W"]
    p = c["points"][0, :, N_CORNER]
    xyz = spec.project_ref(p, c["calib"][0] if c["calib"] is not None else None, c["proj"])
    u, v = xyz[0], xyz[1]
    inside = (u >= -1) & (u <= 1) & (v >= -1) & (v <= 1)
    assert inside.float().mean().item() > 0.9
    ix, iy = ((u + 1) / 2 * (W - 1))[inside], ((v + 1) / 2 * (H - 1))[inside]
    # the texels the bilinear taps read with a nonzero weight
    x1 = torch.where(ix.floor() < ix, ix.floor() + 1, ix.floor()).clamp(max=W - 1).long()
    y1 = torch.where(iy.floor() < iy, iy.floor() + 1, iy.floor()).clamp(max=H - 1).long()
    texels = set((y1 * W + x1).tolist())
    assert H * W - 1 in texels
    tail0 = (H * W - 1) // 128 * 128
    assert sum(t >= tail0 for t in texels) >= min(16, H * W - tail0)


@pytest.mark.parametrize("name", shape_cases())
def test_restatement_matches_reference_shape_golden(name):
    c = load_shape_case(name)
    want = spec.query_ref(c["feat"], c["points"], c["calib"], c["Ws"], c["bs"], c["last_op"], c["proj"])
    assert (want - c["expected"]).abs().max().item() < 2e-6


@pytest.mark.parametrize("name", shape_grad_cases())
def test_grad_restatement_matches_reference_shape_golden(name):
    c = load_shape_grad_case(name)
    _, g64 = query_grad_ref(c["feat"], c["points"], c["calib"], c["Ws"], c["bs"], c["last_op"], c["proj"], dtype=torch.float64)
    assert (g64 - c["grad64"]).abs().max().item() <= 1e-9 * c["grad64"].abs().max().item()
    val, g32 = query_grad_ref(c["feat"], c["points"], c["calib"], c["Ws"], c["bs"], c["last_op"], c["proj"])
    assert (val - c["value"]).abs().max().item() < 2e-6
    ok, msg = within_bar(g32, c["grad32"])
    assert ok, msg


@pytest.mark.parametrize("name", shape_batch_cases())
def test_restatement_per_image_matches_batched_shape_golden(name):
    c = load_shape_batch_case(name)
    assert c["B"] == 3 and c["H"] != c["W"]
    for b in range(c["B"]):
        cal = c["calib"][b:b + 1] if c["calib"] is not None else None
        want = spec.query_ref(c["feat"][b], c["points"][b], cal, c["Ws"], c["bs"], c["last_op"], c["proj"])
        assert (want - c["expected"][b]).abs().max().item() < 2e-6, b


# ---- the kernels on the CPU model --------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return {k: build(tmp_path_factory, "emu_" + k) for k in ("tc", "fp32")}


def _input(c, n, batched=False, res=None, rows=None):
    return dict(feat=c["feat"], rows=c["points"][:, :, :n] if rows is None else rows, calib=c["calib"], proj=c["proj"],
                res=c["chans"][-1] if res is None else res, last_op=c["last_op"], Ws=c["Ws"], bs=c["bs"], batched=batched)


def _run(exe, tmp_path, c, n, batch=None, tag="x", **options):
    """-> [B,Res,n] (a batched launch of B images) or [Res,n] of the query of emu_tc / emu_fp32"""
    res = c["chans"][-1]
    shape = (batch, res, n) if batch else (res, n)
    return run(exe, tmp_path, "query", inp=_input(c, n, batch is not None), shape=shape, options=dict(batch=batch, **options),
               tag=tag)[0]


# 136 points: the 8 border points, the 64-point corner cluster and 64 uniform ones -- three tiles of 64, the last one ragged
TC_CASES = [
    ("g_wide", 136, 1), ("g_wide", 136, 3), ("g_tiny", 136, 1), ("g_tiny", 136, 3), ("g_row", 136, 2), ("g_col", 136, 2),
    pytest.param("g_tall", 136, 1, marks=full_only), pytest.param("g_tall", 136, 3, marks=full_only),
    pytest.param("c_wide", 136, 1, marks=full_only), ("c_wide", 72, 3),
]


@pytest.mark.parametrize("name,n,sms", TC_CASES)
def test_tc_program_matches_reference_shape_golden(emu, tmp_path, name, n, sms):
    c = load_shape_case(name)
    got = _run(emu["tc"], tmp_path, c, n, sms=sms)
    want = c["expected"][:, :n]
    assert (got - want).abs().max().item() <= 1e-4
    assert torch.equal(got[want == 0], want[want == 0]), "out-of-image points must be exactly 0"


@pytest.mark.parametrize("name", shape_batch_cases())
def test_tc_batch_on_non_square_maps(emu, tmp_path, name):
    """B maps of 72 x 136 texels (9792 = 76.5 blocks of 128: each image's G0 ends in a partial block, and image b's blocks
    start at b * 9792 texels) in one launch: within the bar of the batched golden, and image b equal to its B = 1 launch bit
    for bit."""
    c = load_shape_batch_case(name)
    n = 100
    got = _run(emu["tc"], tmp_path, c, n, batch=c["B"], sms=2)
    want = c["expected"][:, :, :n]
    assert (got - want).abs().max().item() <= 1e-4
    assert torch.equal(got[want == 0], want[want == 0])
    for b in range(c["B"]):
        one = dict(c, feat=c["feat"][b:b + 1], points=c["points"][b:b + 1],
                   calib=c["calib"][b:b + 1] if c["calib"] is not None else None)
        assert torch.equal(got[b], _run(emu["tc"], tmp_path, one, n, sms=2, tag="one%d" % b)), b


@pytest.mark.parametrize("name", ["g_wide", "g_tiny"])
def test_g0_products_cover_every_texel(emu, tmp_path, name):
    """The per-texel products of the G0 kernel, the tail block's texels included: G0 = W0f . F against float64 of the same
    fp16 operands (within one fp16 ulp of the result plus the bound of an fp32 sum of C products), the fp16 copy of the map
    exactly, and S4 = W4s . F within the bound of an fp32 sum of C products."""
    c = load_shape_case(name)
    C, H, W = c["feat"].shape[1:]
    M = H * W
    dump = str(tmp_path / "g0.bin")
    _run(emu["tc"], tmp_path, c, 16, sms=2, dump=dump)
    raw = open(dump, "rb").read()
    assert len(raw) == M * 1024 * 2 + M * C * 2 + M * 4
    g0 = np.frombuffer(raw, np.float16, M * 1024).reshape(M, 1024).astype(np.float64)
    f16 = np.frombuffer(raw, np.float16, M * C, offset=M * 1024 * 2).reshape(M, C)
    s4 = np.frombuffer(raw, np.float32, M, offset=M * 1024 * 2 + M * C * 2).astype(np.float64)
    F = c["feat"][0].reshape(C, M).t().numpy()                                   # [texel][C], fp32
    assert np.array_equal(f16.view(np.uint16), F.astype(np.float16).view(np.uint16)), "fp16 copy of the map"
    W0f = c["Ws"][0][:, :C].numpy().astype(np.float16).astype(np.float64)      # [1024][C]
    F16 = F.astype(np.float16).astype(np.float64)
    want = F16 @ W0f.T                                                           # [texel][1024]
    tol = np.spacing(np.abs(want).astype(np.float16)).astype(np.float64) + (C + 2) * 2.0 ** -24 * (np.abs(F16) @ np.abs(W0f.T))
    bad = np.abs(g0 - want) > tol
    assert not bad.any(), "G0 off at %d entries, first texel %d of %d" % (bad.sum(), np.argwhere(bad)[0][0], M)
    W4s = c["Ws"][4][:, 128:128 + C].numpy().astype(np.float64)                 # layer 4 input: [hidden 128, C features, z]
    exact = F.astype(np.float64) @ W4s[0]
    bound = (C + 2) * 2.0 ** -24 * (np.abs(F.astype(np.float64)) @ np.abs(W4s[0]))
    assert (np.abs(s4 - exact) <= bound).all(), np.abs(s4 - exact).max()


FP32_CASES = [("g_wide", 136), ("g_tall", 136), ("g_tiny", 136), ("g_row", 136), ("g_col", 136), ("c_wide", 72),
              pytest.param("g_limit", 136, marks=full_only), pytest.param("g_over", 136, marks=full_only),
              pytest.param("c_over", 72, marks=full_only)]


@pytest.mark.parametrize("name,n", FP32_CASES)
def test_fp32_kernel_matches_reference_shape_golden(emu, tmp_path, name, n):
    c = load_shape_case(name)
    got = _run(emu["fp32"], tmp_path, c, n)
    want = c["expected"][:, :n]
    ok, msg = within_fp32_bar(got, dict(c, expected=want, expected64=c["expected64"][:, :n]))
    assert ok, msg
    assert torch.equal(got[want == 0], want[want == 0]), "out-of-image points must be exactly 0"


@pytest.mark.parametrize("name", shape_grad_cases())
def test_grad_kernel_matches_reference_shape_golden(emu, tmp_path, name):
    """the point gradient within its bar of the reference's fp32 autograd, and its value the fp32 query's bit for bit"""
    c = load_shape_grad_case(name)
    n = 136
    out, _ = run(emu["fp32"], tmp_path, "grad", inp=_input(c, n, res=1), shape=(4 * n,), options=dict(sms=3), tag="g")
    val, dp = out[:n].reshape(1, n), out[n:].reshape(3, n)
    assert (val - c["value"][:, :n]).abs().max().item() <= 2e-5
    ok, msg = within_bar(dp, c["grad32"][:, :n])
    assert ok, msg
    assert torch.equal(val, _run(emu["fp32"], tmp_path, c, n, tag="q"))


# ---- the colour surface render on a non-square map ------------------------------------------------------------------------
R_CANVAS = 65


@pytest.mark.parametrize("program", ["tc", "fp32"])
def test_colour_surface_render_on_a_non_square_map(emu, tmp_path, program):
    """colorization() of 120 visible vertices through the colour head on the 88 x 120 map, by the tensor-core render and by
    its exact fp32 twin, against the restatement driven by the oracle's query."""
    c = load_shape_case("c_wide")
    g = torch.Generator().manual_seed(9)
    n = 120
    cols = torch.randperm(R_CANVAS * R_CANVAS, generator=g)[:n]
    X, Y = cols // R_CANVAS, cols % R_CANVAS
    Z = torch.rand(n, generator=g) * (R_CANVAS - 1)
    rows = torch.stack([X.float(), Y.float(), Z])[None]
    got, _ = run(emu[program], tmp_path, "surface", R_CANVAS, n, -1, -1, -1, 1, 1, 1,        # the render box [b_min, b_max]
                 inp=_input(c, n, res=3, rows=rows), shape=(R_CANVAS, R_CANVAS, 3), options=dict(sms=2))

    def query_c(points, calib):
        return spec.query_ref(c["feat"], points, calib, c["Ws"], c["bs"], spec.LAST_TANH)

    want = spec.colorization_ref(query_c, X, Y, Z, c["calib"], resolution=R_CANVAS)
    assert (got - want).abs().max().item() <= (1e-4 if program == "tc" else 2e-5)
    untouched = torch.ones(R_CANVAS, R_CANVAS, dtype=torch.bool)
    untouched[X, Y] = False
    assert bool((got[untouched] == 1.0).all())
