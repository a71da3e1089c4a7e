"""CPU tier of the captured colour frame: the surface render of both query programs (the colour head's tensor-core program
and its exact fp32 twin) and the normal-image kernel, compiled unmodified against the CPU emulation layer (tests/emu), with
the vertex count on the device and the range guard decided there; and the compiler report of the new fp32 instantiations."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from oracle import spec
from emu_harness import build, needs_emu, ptxas_report, run

pytestmark = needs_emu

R = 65
UNIT = ((-1.0, -1.0, -1.0), (1.0, 1.0, 1.0))
B1 = ((-0.83, -1.17, -0.61), (0.91, 1.06, 0.77))     # asymmetric, no power-of-two extent: the axes cannot stand in for each other


@pytest.fixture(scope="module")
def emu_tc(tmp_path_factory):
    return build(tmp_path_factory, "emu_tc")


@pytest.fixture(scope="module")
def emu_fp32(tmp_path_factory):
    return build(tmp_path_factory, "emu_fp32")


@pytest.fixture(scope="module")
def emu_normals(tmp_path_factory):
    return build(tmp_path_factory, "emu_render_normals")


@pytest.fixture(scope="module")
def scene():
    """The colour head, a 32 x 32 colour map, and 200 visible vertices on distinct (x, y) columns of an R = 65 canvas."""
    Ws, bs = spec.make_weights(spec.C_CHANNELS, 77)
    feat = spec.make_feat(512, 32, 32, 78)
    cal = spec.scene_calib(20, 33)
    g = torch.Generator().manual_seed(7)
    cols = torch.randperm(R * R, generator=g)[:200]
    X, Y = cols // R, cols % R
    Z = torch.rand(200, generator=g) * (R - 1)
    return dict(Ws=Ws, bs=bs, feat=feat, cal=cal, X=X, Y=Y, Z=Z)


def _input(sc, rows, feat=None):
    """the harnesses' in.bin: the colour head and map, three rows of N floats"""
    return dict(feat=sc["feat"] if feat is None else feat, rows=rows, calib=sc["cal"], proj="orthogonal", res=3,
                last_op=spec.LAST_TANH, Ws=sc["Ws"], bs=sc["bs"])


def _vertex_rows(sc, n=200):
    return torch.stack([sc["X"][:n].float(), sc["Y"][:n].float(), sc["Z"][:n]]).numpy()


def _box_args(box):
    return ["%.9g" % np.float32(v) for v in box[0] + box[1]]


def _fp32_surface(exe, tmp_path, sc, count, sms=3, n=200, feat=None, box=UNIT, **options):
    return run(exe, tmp_path, "surface", R, count, *_box_args(box), inp=_input(sc, _vertex_rows(sc, n), feat), shape=(R, R, 3),
               options=dict(sms=sms, **options))[0]


def _tc_surface(exe, tmp_path, sc, count, sms=2, n=200, host=False, feat=None, box=UNIT, **options):
    img, r = run(exe, tmp_path, "surface", R, count, *_box_args(box), inp=_input(sc, _vertex_rows(sc, n), feat),
                 shape=(R, R, 3), options=dict(sms=sms, eager=host, print_amax=True, **options))
    return img, float(r.stdout.split()[0])


def _want(sc, n=200, box=UNIT):
    def query_c(points, calib):
        return spec.query_ref(sc["feat"], points, calib, sc["Ws"], sc["bs"], spec.LAST_TANH)
    return spec.colorization_ref(query_c, sc["X"][:n], sc["Y"][:n], sc["Z"][:n], sc["cal"], resolution=R, b_min=box[0],
                                 b_max=box[1])


# ---- the exact fp32 render ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sms,box", [pytest.param(1, UNIT, id="1"), pytest.param(3, UNIT, id="3"), pytest.param(3, B1, id="3-B1")])
def test_exact_surface_render_matches_restatement(emu_fp32, tmp_path, scene, sms, box):
    """colorization (RTL/main.py:212-249) with the exact kernel: within the fp32 query bar of the restatement driven by the
    oracle's query, and pixels without a vertex keep the canvas colour."""
    got = _fp32_surface(emu_fp32, tmp_path, scene, 200, sms=sms, box=box)
    want = _want(scene, box=box)
    assert (got - want).abs().max().item() <= 2e-5
    untouched = torch.ones(R, R, dtype=torch.bool)
    untouched[scene["X"], scene["Y"]] = False
    assert bool((got[untouched] == 1.0).all())


def test_exact_surface_render_is_the_rows_query_plus_scatter(emu_fp32, tmp_path, scene):
    """Bit for bit: the fused render = the exact ROWS query on world points made with the same two fp32 roundings per axis
    (index * (b_max - b_min) / R, then + b_min), followed by the same scatter of v * 0.5 + 0.5 -- over the unit cube and a
    box whose three extents differ."""
    for box in (UNIT, B1):
        got = _fp32_surface(emu_fp32, tmp_path, scene, 200, box=box)
        f32 = np.float32
        lo, hi = np.asarray(box[0], f32), np.asarray(box[1], f32)
        scale = ((hi - lo) / f32(R)).astype(f32)[:, None]
        v = _vertex_rows(scene).astype(f32)
        v[2] = f32(R) - v[2]
        world = (v * scale).astype(f32) + lo[:, None]
        vals = run(emu_fp32, tmp_path, "query", inp=_input(scene, world), shape=(3, 200), tag="w")[0].numpy()
        want = np.ones((R, R, 3), f32)
        want[scene["X"].numpy(), scene["Y"].numpy(), :] = ((vals * f32(0.5)).astype(f32) + f32(0.5)).T
        assert np.array_equal(got.numpy().view(np.int32), want.view(np.int32)), box


def test_exact_surface_render_device_count(emu_fp32, tmp_path, scene):
    """The count lives on the device: vertices at or beyond it are neither evaluated nor drawn (the tail of the buffers holds
    valid vertices, whose pixels must keep the background), a count of 0 leaves the canvas untouched, and a count above the
    capacity is clamped to it."""
    n = 120
    got = _fp32_surface(emu_fp32, tmp_path, scene, 90, n=n, canvas_bg=0.25)
    full = _fp32_surface(emu_fp32, tmp_path, scene, n, n=n, canvas_bg=0.25)
    X, Y = scene["X"], scene["Y"]
    assert torch.equal(got[X[:90], Y[:90]], full[X[:90], Y[:90]])
    assert bool((got[X[90:n], Y[90:n]] == 0.25).all()) and bool((full[X[90:n], Y[90:n]] != 0.25).all())
    assert bool((_fp32_surface(emu_fp32, tmp_path, scene, 0, n=n) == 1.0).all())
    assert torch.equal(_fp32_surface(emu_fp32, tmp_path, scene, 10 ** 9, n=n, canvas_bg=0.25), full)


@pytest.mark.parametrize("limit,writes", [("1.0", True), ("100.0", False)])
def test_exact_surface_render_guard_sense(emu_fp32, tmp_path, scene, limit, writes):
    """MP_GUARD_OUT_OF_RANGE: the exact twin renders a frame whose max |feature| (here 5) is above the head's limit and
    leaves the canvas of an in-range frame to the tensor-core launch."""
    got = _fp32_surface(emu_fp32, tmp_path, scene, 40, n=40,
                        guard="out", limit=limit, amax=5.0)
    assert bool((got == 1.0).all()) != writes


# ---- the tensor-core render with the count on the device ---------------------------------------------------------------
def test_tc_surface_render_device_count_equals_host_count(emu_tc, tmp_path, scene):
    """The render of a captured step (count read on the device, capacity n) equals the eager launch given the same count on
    the host, bit for bit, over the unit cube and a box whose three extents differ; vertices past the count keep the
    background, and a count above the capacity is clamped."""
    n, k = 130, 100
    X, Y = scene["X"], scene["Y"]
    for box in (B1, UNIT):
        dev, _ = _tc_surface(emu_tc, tmp_path, scene, k, n=n, canvas_bg=0.25, box=box)
        host, _ = _tc_surface(emu_tc, tmp_path, scene, k, n=n, host=True, canvas_bg=0.25, box=box)
        assert torch.equal(dev, host)
        assert bool((dev[X[k:n], Y[k:n]] == 0.25).all())
        assert (dev[X[:k], Y[:k]] - _want(scene, k, box)[X[:k], Y[:k]]).abs().max().item() <= 1e-4, box
    clamped, _ = _tc_surface(emu_tc, tmp_path, scene, 10 ** 9, n=n, canvas_bg=0.25)
    host_all, _ = _tc_surface(emu_tc, tmp_path, scene, n, n=n, host=True, canvas_bg=0.25)
    assert torch.equal(clamped, host_all)
    zero, _ = _tc_surface(emu_tc, tmp_path, scene, 0, n=n)
    assert bool((zero == 1.0).all())


@pytest.mark.parametrize("limit,writes", [("0.01", False), ("100.0", True)])
def test_tc_surface_render_guard_sense(emu_tc, tmp_path, scene, limit, writes):
    """MP_GUARD_IN_RANGE: the tensor-core launch renders a frame whose max |feature| is inside the head's limit and leaves
    the canvas of a frame above it untouched (the exact twin renders that one)."""
    got, amax = _tc_surface(emu_tc, tmp_path, scene, 40, n=40, guard="in", limit=limit)
    assert abs(amax - scene["feat"].abs().max().item()) <= 1e-6 * amax
    assert bool((got == 1.0).all()) != writes


# ---- the normal image --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("count,blocks", [(300, 1), (250, 2), (0, 1), (10 ** 6, 3)])
def test_normal_image_is_torchs(emu_normals, tmp_path, count, blocks):
    """canvas[X, Y] = clamp((norm + 1) / 2, 0, 1) for the vertices below the device-side count, bit for bit what
    colorization(norm=...) gives in torch -- NaN normals stay NaN, values outside [-1, 1] are clamped."""
    Rn, cap = 33, 300
    g = torch.Generator().manual_seed(11)
    cols = torch.randperm(Rn * Rn, generator=g)[:cap]
    X, Y = cols // Rn, cols % Rn
    N = (torch.rand(cap, 3, generator=g) * 3 - 1.5).float()
    N[::7, 1] = float("nan")
    N[5] = float("nan")
    fin, fout = str(tmp_path / "n.bin"), str(tmp_path / "n.f32")
    with open(fin, "wb") as f:
        f.write(X.numpy().astype(np.int64).tobytes())
        f.write(Y.numpy().astype(np.int64).tobytes())
        f.write(N.numpy().tobytes())
    r = subprocess.run([os.path.join(emu_normals), str(Rn), str(cap), str(count), str(blocks), fin, fout], capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    got = np.fromfile(fout, dtype=np.float32).reshape(Rn, Rn, 3)
    k = min(count, cap)
    want = spec.colorization_ref(None, X[:k], Y[:k], None, None, resolution=Rn, norm=N[:k]).numpy()
    assert k == 0 or np.isnan(want).any()
    assert np.array_equal(got.view(np.int32), want.view(np.int32))


# ---- compiler report of the exact program -----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def fp32_ptxas():
    """{(tile P, surface instantiation): its ptxas lines} of query_fp32_kernel"""
    stats = {}
    for name, lines in ptxas_report("query_fp32.cu")[0]:
        m = re.search(r"query_fp32_kernelILi(\d+)ELb([01])E", name)
        if m:
            stats[(int(m.group(1)), m.group(2) == "1")] = " ".join(lines)
    return stats


def test_fp32_surface_instantiations_do_not_spill(fp32_ptxas):
    for P in (8, 16, 32):
        s = fp32_ptxas[(P, True)]
        assert "0 bytes spill stores, 0 bytes spill loads" in s, s


def test_fp32_query_instantiations_keep_their_report(fp32_ptxas):
    """The query instantiations are untouched by the surface source: same registers, same 104-byte frame, no spill."""
    for P, regs in ((8, 102), (16, 125), (32, 145)):
        s = fp32_ptxas[(P, False)]
        assert "104 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in s, s
        assert "Used %d registers" % regs in s, s
