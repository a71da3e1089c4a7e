"""CPU-side checks of the integer / byte CUDA kernels: the kernel sources (monoport_b200/csrc/*_kernels.cuh, mp_scan.cuh)
are compiled UNMODIFIED against tests/emu/cuda_emu.h (one OS thread per CUDA thread, barriers for __syncthreads and
warp shuffles) and compared with the oracle.  The build container has no GPU; this catches indexing / scan / table
mistakes before a kernel is sent to an H100.  The `-m gpu` tests remain the parity tests of the real library."""
import os
import subprocess

import numpy as np
import pytest

from oracle import spec
from emu_harness import build, needs_gxx, write_input

pytestmark = needs_gxx
# one OS thread per CUDA thread is slow: the heaviest cases only run with MONOPORT_B200_EMU_FULL=1 (they pass; the default
# set keeps the CPU tier at a few minutes)
FULL = os.environ.get("MONOPORT_B200_EMU_FULL", "0") == "1"
full_only = pytest.mark.skipif(not FULL, reason="heavy emulation case: set MONOPORT_B200_EMU_FULL=1")


@pytest.fixture(scope="module")
def emu_mcubes(tmp_path_factory):
    return build(tmp_path_factory, "emu_mcubes")


def _run_mcubes(exe, vol, tmp_path, iso=0.5):
    D, H, W = vol.shape
    vin, vout, fout = (str(tmp_path / n) for n in ("vol.f32", "verts.f32", "faces.i32"))
    np.ascontiguousarray(vol, dtype=np.float32).tofile(vin)
    r = subprocess.run([exe, str(D), str(H), str(W), repr(float(iso)), vin, vout, fout], capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr
    nv, nf = (int(x) for x in r.stdout.split())
    v = np.fromfile(vout, dtype=np.float32).reshape(-1, 3)
    f = np.fromfile(fout, dtype=np.int32).reshape(-1, 3)
    assert v.shape[0] == nv and f.shape[0] == nf
    return v, f


@pytest.mark.parametrize("kind,R,iso", [
    pytest.param("sphere", 33, 0.5, id="sphere-33"), pytest.param("ellipsoid", 40, 0.5, id="ellipsoid-40"),
    pytest.param("two_blobs", 49, 0.5, id="two_blobs-49"), pytest.param("steps", 33, 0.5, id="steps-33"),
    pytest.param("steps", 33, 0.25, id="steps-33-iso0.25"), pytest.param("corner", 33, 0.5, id="corner-33"),
    pytest.param("ball01", 17, 0.5, id="ball01-17")])
def test_mcubes_kernels_match_oracle_on_analytic_volumes(emu_mcubes, tmp_path, kind, R, iso):
    """steps: nodes equal to the iso value (not inside: t = 0 or 1 on the edge); corner / ball01: cut by the box faces."""
    vol = spec.analytic_volume(R, kind)
    V, F = spec.marching_cubes_ref(vol, iso)
    v, f = _run_mcubes(emu_mcubes, vol, tmp_path, iso)
    assert len(F) > 0
    assert np.array_equal(f, F), "topology must be bit-exact"
    assert v.shape == V.shape and np.array_equal(v, V)
    if kind == "sphere":
        # independent of the restatement: the field is 0.5 + 4 (0.6 - |p|), so every vertex must sit on the sphere of radius
        # 0.6 up to the error of interpolating |p| linearly along a grid edge (h^2 / 8r), and the mesh must be closed
        p = (v + 0.5) / R * 2.0 - 1.0
        assert np.abs(np.linalg.norm(p, axis=1) - 0.6).max() < (2.0 / R) ** 2 / (8 * 0.6) * 1.5
        e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]).astype(np.int64)
        key, rkey = e[:, 0] * len(v) + e[:, 1], e[:, 1] * len(v) + e[:, 0]
        assert len(np.unique(key)) == len(key) and np.array_equal(np.sort(key), np.sort(rkey))       # closed, consistently oriented
        assert len(v) - len(np.unique(np.minimum(key, rkey))) + len(f) == 2                          # Euler characteristic of a sphere


@pytest.mark.parametrize("shape", [(20, 17, 23), (9, 40, 35), (2, 2, 2), (3, 70, 2), (3, 5, 131), (2, 3, 257), (2, 9, 128),
                                   (2, 2, 33)])
def test_mcubes_kernels_match_oracle_on_noise(emu_mcubes, tmp_path, shape):
    """Dense noise: nearly every node is active (full shared-memory queues, every table case), odd and tiny shapes
    (rows shorter than a warp, rows of 2^k+1 nodes whose last chunk holds one node, rows longer than one chunk group,
    row tiles hanging over H, scan chunks hanging over n)."""
    vol = np.random.default_rng(sum(shape)).random(shape, dtype=np.float32)
    V, F = spec.marching_cubes_ref(vol)
    v, f = _run_mcubes(emu_mcubes, vol, tmp_path)
    assert np.array_equal(f, F.reshape(-1, 3))
    assert v.shape == V.shape and np.array_equal(v, V)


@pytest.mark.parametrize("fill", [0.0, 1.0])
def test_mcubes_kernels_empty_volume(emu_mcubes, tmp_path, fill):
    v, f = _run_mcubes(emu_mcubes, np.full((9, 9, 9), fill, dtype=np.float32), tmp_path)
    assert v.shape[0] == 0 and f.shape[0] == 0


# ---- the ordered scan itself (mp_scan.cuh): exclusive prefixes of two packed counters -----------------------------------
@pytest.fixture(scope="module")
def emu_scan(tmp_path_factory):
    return build(tmp_path_factory, "emu_scan")


@pytest.mark.parametrize("vec", [0, 1])
@pytest.mark.parametrize("n", [0, 1, 7, 8, 9, 2047, 2048, 2049, 70001])
def test_ordered_scan_matches_cumsum(emu_scan, tmp_path, n, vec):
    _check_scan(emu_scan, tmp_path, n, vec)


@full_only
def test_ordered_scan_many_ctas(emu_scan, tmp_path):
    """More CTA totals than threads in the last CTA: every thread of it owns a run of several totals."""
    _check_scan(emu_scan, tmp_path, 2048 * 256 + 4097, 1)


def _check_scan(exe, tmp_path, n, vec):
    rng = np.random.default_rng(n + vec)
    b = (rng.integers(0, 64, size=n, dtype=np.uint8) * (rng.random(n) < 0.3)).astype(np.uint8)
    fin, fout = str(tmp_path / "in.u8"), str(tmp_path / "out.u64")
    b.tofile(fin)
    r = subprocess.run([exe, str(n), str(vec), fin, fout], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    lo, hi = (b & 7).astype(np.uint64), (b >> 3).astype(np.uint64)
    assert [int(x) for x in r.stdout.split()] == [int(lo.sum()), int(hi.sum())]
    if n:
        want = (np.cumsum(lo) - lo) + ((np.cumsum(hi) - hi) << np.uint64(32))
        assert np.array_equal(np.fromfile(fout, dtype=np.uint64), want)


# ---- coarse-to-fine engine kernels (octree_kernels.cuh) against the restatement: volume AND evaluated node lists --------
@pytest.fixture(scope="module")
def emu_octree(tmp_path_factory):
    return build(tmp_path_factory, "emu_octree")


def _run_octree(exe, tmp_path, mode, field, res, kpts=None, balance=0.5):
    fin, fvol, fidx = (str(tmp_path / n) for n in ("dense.f32", "vol.f32", "idx.i32"))
    np.ascontiguousarray(field, dtype=np.float32).tofile(fin)
    args = [exe, mode, repr(float(balance)), fin, fvol, fidx, str(len(res))] + [str(r) for r in res] + [str(k) for k in (kpts or [])]
    r = subprocess.run(args, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr
    out = [int(x) for x in r.stdout.split()]
    vol = np.fromfile(fvol, dtype=np.float32)
    return out[0], out[1:], vol, np.fromfile(fidx, dtype=np.int32)


@pytest.mark.parametrize("mode,field_kind,res,balance", [
    pytest.param("faster", "sphere", [9, 17, 33, 65], 0.5, id="faster-sphere-res0"),
    pytest.param("faster", "two_blobs", [5, 9, 17, 33, 65], 0.5, id="faster-two_blobs-res1"),
    pytest.param("faster", "ellipsoid", [9, 17, 33], 0.5, id="faster-ellipsoid-res2"),
    pytest.param("lossless", "two_blobs", [9, 17, 33], 0.5, marks=full_only, id="lossless-two_blobs-res3"),
    pytest.param("lossless", "sphere", [9, 17], 0.5, id="lossless-sphere-res4"),
    pytest.param("topk", "sphere", [9, 17, 33], 0.5, marks=full_only, id="topk-sphere-res5"),
    pytest.param("topk", "sphere", [9, 17], 0.5, id="topk-sphere-res6"),
    # fields that reach the box (clamped dilation boxes with mixed neighbourhoods), nodes equal to the balance, other balances
    ("lossless", "noise", [5, 9, 17], 0.3), ("lossless", "noise", [5, 9, 17], 0.7), ("faster", "noise", [5, 9, 17, 33], 0.3),
    ("faster", "corner", [9, 17, 33], 0.5), ("faster", "slab", [9, 17, 33], 0.7), ("faster", "steps", [5, 9, 17, 33], 0.5),
    ("lossless", "corner", [9, 17], 0.3), ("lossless", "steps", [9, 17], 0.5), ("lossless", "slab", [5, 9, 17], 0.7),
    ("lossless", "ball01", [5, 9, 17], 0.5), ("topk", "noise", [5, 9, 17], 0.3), ("topk", "steps", [9, 17], 0.5),
    ("topk", "corner", [9, 17], 0.7)])
def test_octree_kernels_match_restatement(emu_octree, tmp_path, mode, field_kind, res, balance):
    import torch
    from helpers import lookup_query
    R = res[-1]
    field = spec.analytic_volume(R, field_kind)
    fn_o, _ = lookup_query(torch.from_numpy(field))
    kpts = [0, 1500, 5000][:len(res)] if mode == "topk" else None
    if mode == "topk":
        want, stats = spec.seg3d_topk_ref(fn_o, res, kpts, balance=balance, return_stats=True)
    else:
        want, stats = spec.seg3d_lossless_ref(fn_o, res, balance=balance, faster=(mode == "faster"), return_stats=True)
    nonempty, counts, vol, idx = _run_octree(emu_octree, tmp_path, mode, field, res, kpts, balance)
    assert nonempty == 1 and want is not None
    assert counts == [int(s["idx"].numel()) for s in stats]
    assert np.array_equal(vol.reshape(R, R, R), want.numpy()), "volume must be bit-identical to the restatement"
    assert np.array_equal(idx, np.concatenate([s["idx"].numpy().astype(np.int32) for s in stats])), "node lists / order"


def test_octree_kernels_empty_field(emu_octree, tmp_path):
    """Level 0 finds nothing occupied: the levels still run (no host read of the flag, as in a captured frame) but evaluate
    nothing -- also the top-k levels, whose node count is gated on the device-side flag."""
    for mode in ("faster", "lossless", "topk"):
        kpts = [0, 100, 2000] if mode == "topk" else None
        nonempty, counts, vol, idx = _run_octree(emu_octree, tmp_path, mode, np.zeros((33, 33, 33), np.float32), [9, 17, 33],
                                                 kpts)
        assert nonempty == 0 and counts[0] == 729 and sum(counts[1:]) == 0 and vol.size == 0, mode


# ---- visible-surface kernels (surface_kernels.cuh) against the goldens produced by the unmodified RTL/recon.py -------------
@pytest.fixture(scope="module")
def emu_surface(tmp_path_factory):
    return build(tmp_path_factory, "emu_surface")


@pytest.mark.parametrize("golden", ["fv_sphere_33", "fv_two_blobs_65", "fv_ellipsoid_65"] + [
    "fv_%s_%d" % (k, R) for k in ("corner", "slab", "ball01", "noise") for R in (33, 65)])
def test_surface_kernels_match_reference_golden(emu_surface, tmp_path, golden_dir, golden):
    g = np.load(os.path.join(golden_dir, golden + ".npz"))
    R = int(g["R"])
    fin, fout = str(tmp_path / "vol.f32"), str(tmp_path / "out.bin")
    spec.analytic_volume(R, str(g["kind"])).tofile(fin)
    for di, d in enumerate(("front", "back", "left", "right")):
        r = subprocess.run([emu_surface, str(R), str(di), fin, fout], capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr
        k = int(r.stdout)
        raw = open(fout, "rb").read()
        X = np.frombuffer(raw[:8 * k], dtype=np.int64)
        Y = np.frombuffer(raw[8 * k:16 * k], dtype=np.int64)
        Z = np.frombuffer(raw[16 * k:20 * k], dtype=np.float32)
        N = np.frombuffer(raw[20 * k:32 * k], dtype=np.float32).reshape(-1, 3)
        assert np.array_equal(X, g["X_" + d]) and np.array_equal(Y, g["Y_" + d])
        np.testing.assert_allclose(Z, g["Z_" + d], rtol=0, atol=1e-5, equal_nan=True)
        np.testing.assert_allclose(N, g["N_" + d], rtol=0, atol=1e-6, equal_nan=True)


# ---- the flagship kernels: query_tc.cu (weight packing, launch logic, G0 GEMM kernel, fused wgmma sample+MLP program) on
#      the functional model of the wgmma / mbarrier / bulk-copy layer (tests/emu/tc_ptx_emu.h), with asynchronous operations
#      deferred adversarially, against the goldens of the UNMODIFIED reference ---------------------------------------------
@pytest.fixture(scope="module")
def emu_query_tc(tmp_path_factory):
    return build(tmp_path_factory, "emu_query_tc")


def _run_query_tc(exe, tmp_path, case, n, program, sms, extra_env=None):
    import torch
    res = case["expected"].shape[0]
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.f32")
    write_input(fin, case["feat"], case["points"][:, :, :n], case["calib"], case["proj"], res, case["last_op"], case["Ws"],
                case["bs"])
    env = dict(os.environ)
    env.update(extra_env or {})
    r = subprocess.run([exe, fin, fout, str(program), str(sms)], capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0, r.stderr[-2000:]
    return torch.from_numpy(np.fromfile(fout, dtype=np.float32)).reshape(res, n)


@pytest.mark.parametrize("name,n,program,sms", [
    ("g_smallmap", 300, 3, 1),      # one CTA walks five tiles: the weight ring across tiles, ragged last tile
    ("g_smallmap", 300, 3, 2),      # two CTAs
    ("g_smallmap", 200, 103, 1),    # program v3 with the fused slab exchange (peer stores)
    pytest.param("g_rot33", 130, 3, 132, marks=full_only),   # 128 x 128 map: 128 CTAs of the G0 GEMM, rotated calibration
    ("g_persp", 100, 3, 1),         # perspective projection
    ("g_nocalib", 150, 3, 3),       # calibs=None
])
def test_tcgen05_kernels_match_reference_golden(emu_query_tc, tmp_path, name, n, program, sms):
    from helpers import load_query_case
    case = load_query_case(name)
    got = _run_query_tc(emu_query_tc, tmp_path, case, n, program, sms)
    err = (got - case["expected"][:, :n]).abs().max().item()
    assert err <= 1e-4, err          # the GPU parity bar for the tensor-core programs (measured on the model: ~2e-5)


@pytest.mark.parametrize("name,n,program,sms", [
    ("g_smallmap", 300, 3, 1),      # geometry head, one CTA walks all five tiles: the weight ring wraps across tiles
    ("g_smallmap", 300, 3, 2),      # two CTAs
    ("g_smallmap", 200, 103, 3),    # with the peer stores of the fused slab exchange
    ("c_rot33", 200, 0, 1),         # colour head: two-stage ring, (hi, lo) pass of layer 3
])
@pytest.mark.parametrize("order", ["random:1", "random:2", "random:3"])
def test_tcgen05_handoffs_survive_other_completion_orders(emu_query_tc, tmp_path, name, n, program, sms, order):
    """The model completes queued bulk copies in issue order by default.  The hand-off protocol (weight ring, operand
    buffers, wgmma groups) must not depend on that: random completion orders of the copies give the same bits, for both
    heads and for one or several CTAs."""
    import torch
    from helpers import load_query_case
    case = load_query_case(name)
    want = _run_query_tc(emu_query_tc, tmp_path, case, n, program, sms)
    got = _run_query_tc(emu_query_tc, tmp_path, case, n, program, sms, dict(EMU_TC_ORDER=order))
    assert torch.equal(got, want)
    assert (got - case["expected"][:, :n]).abs().max().item() <= 1e-4


@pytest.mark.parametrize("order", ["copies", "random:3"])
def test_tcgen05_colour_head_matches_reference_golden(emu_query_tc, tmp_path, order):
    """PIFuNetCMLP (513 -> 3, Tanh, 512-channel map): the 512-channel skip operand, the (hi, lo) pass of layer 3, eight-K-block
    G0 GEMM, three fp32 last-layer outputs; one emulated SM walks all four tiles (default completion order of the bulk
    copies and a random one)."""
    from helpers import load_query_case
    case = load_query_case("c_rot33")
    n = 200
    got = _run_query_tc(emu_query_tc, tmp_path, case, n, 0, 1, {"EMU_TC_ORDER": order})
    err = (got - case["expected"][:, :n]).abs().max().item()
    assert err <= 1e-4, err
    zero = case["expected"][:, :n] == 0
    assert (got[zero] == 0).all(), "out-of-image points must be exactly 0"


def _write_tc_input(path, case, n):
    """n points at the origin (the grid and node-list sources make their own)"""
    write_input(path, case["feat"], np.zeros((3, n)), case["calib"], "orthogonal", 1, case["last_op"], case["Ws"], case["bs"])


@pytest.mark.parametrize("program", [3, 103])
def test_tcgen05_kernels_grid_source(emu_query_tc, tmp_path, program):
    """mp_query_grid's point source: node centres of a z slab generated in-kernel (103: also stored into the peer volumes
    at the slab's offset, the fused slab exchange)."""
    import torch
    from helpers import load_query_case
    case = load_query_case("g_smallmap")
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.f32")
    _write_tc_input(fin, case, 4)
    R, z0, nz = 13, 3, 5
    r = subprocess.run([emu_query_tc, fin, fout, str(program), "2", "grid", str(R), str(z0), str(nz)], capture_output=True,
                       text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    got = torch.from_numpy(np.fromfile(fout, dtype=np.float32))
    pts = spec.level_points(spec._grid_coords(R, 1), R, (-1, -1, -1), (1, 1, 1))[z0 * R * R:(z0 + nz) * R * R].t().contiguous()
    want = spec.query_ref(case["feat"], pts, case["calib"], case["Ws"], case["bs"], spec.LAST_SIGMOID)[0]
    assert got.numel() == nz * R * R and (got - want).abs().max().item() <= 1e-4


@pytest.mark.parametrize("program", [3])
def test_tcgen05_kernels_node_list_source(emu_query_tc, tmp_path, program):
    """The octree engine's fused path: an index list with a device-side count below the list capacity, values scattered
    into the level volume; nodes that are not on the list stay untouched."""
    import torch
    from helpers import load_query_case
    case = load_query_case("g_smallmap")
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.f32")
    _write_tc_input(fin, case, 4)
    R, res = 33, 9
    r = subprocess.run([emu_query_tc, fin, fout, str(program), "3", "nodes", str(R), str(res)], capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    got = torch.from_numpy(np.fromfile(fout, dtype=np.float32))
    idx = torch.arange(0, res ** 3, 3)
    cc = torch.stack([idx % res, (idx // res) % res, idx // (res * res)], 1) * ((R - 1) // (res - 1))
    pts = spec.level_points(cc, R, (-1, -1, -1), (1, 1, 1)).t().contiguous()
    want = torch.full((res ** 3,), -4242.0)
    want[idx] = spec.query_ref(case["feat"], pts, case["calib"], case["Ws"], case["bs"], spec.LAST_SIGMOID)[0]
    assert (got - want).abs().max().item() <= 1e-4
    assert bool((got[want == -4242.0] == -4242.0).all())


@pytest.mark.parametrize("kind,world", [("nodes", 2), ("nodes", 3), ("grid", 2)])
def test_tcgen05_list_sharding_is_bit_identical(emu_query_tc, tmp_path, kind, world):
    """Multi-GPU list sharding of a query (octree levels, balanced dense ranges): `world` launches, launch r evaluating the
    r-th 128-aligned window of the point list -- also through the peer stores -- reproduce the unsharded launch bit for
    bit (243 nodes over 2 / 3 windows incl. an empty one; 5*13*13 grid nodes over 2)."""
    from helpers import load_query_case
    case = load_query_case("g_smallmap")
    fin = str(tmp_path / "in.bin")
    _write_tc_input(fin, case, 4)
    args = ["nodes", "33", "9"] if kind == "nodes" else ["grid", "13", "3", "5"]
    outs = []
    for w in (1, world):
        fout = str(tmp_path / ("w%d.f32" % w))
        r = subprocess.run([emu_query_tc, fin, fout, "103", "2"] + args, capture_output=True, text=True, timeout=900,
                           env=dict(os.environ, EMU_SHARD_WORLD=str(w)))
        assert r.returncode == 0, r.stderr[-2000:]
        outs.append(np.fromfile(fout, dtype=np.float32))
    assert outs[0].size > 0 and np.array_equal(outs[0], outs[1])


def test_tcgen05_colour_head_fused_surface_rendering(emu_query_tc, tmp_path):
    """mp_colorize_surface: visible-surface vertices (X, Y, R - Z) -> world (mat_color) -> netC -> pred*0.5+0.5 -> canvas, one
    launch, against the restatement of RTL/main.py:212-249 driven by the oracle's query (32 x 32 colour map)."""
    import torch
    Ws, bs = spec.make_weights(spec.C_CHANNELS, 77)
    feat = spec.make_feat(512, 32, 32, 78)
    cal = spec.scene_calib(20, 33)
    R, n = 65, 200
    g = torch.Generator().manual_seed(7)
    cols = torch.randperm(R * R, generator=g)[:n]                     # at most one vertex per (x, y) column
    X, Y = cols // R, cols % R
    Z = torch.rand(n, generator=g) * (R - 1)
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.f32")
    write_input(fin, feat, torch.stack([X.float(), Y.float(), Z]), cal, "orthogonal", 3, spec.LAST_TANH, Ws, bs)
    r = subprocess.run([emu_query_tc, fin, fout, "0", "2", "surface", str(R)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    got = torch.from_numpy(np.fromfile(fout, dtype=np.float32)).reshape(R, R, 3)

    def query_c(points, calib):
        return spec.query_ref(feat, points, calib, Ws, bs, spec.LAST_TANH)

    want = spec.colorization_ref(query_c, X, Y, Z, cal, resolution=R)
    assert (got - want).abs().max().item() <= 1e-4
    untouched = torch.ones(R, R, dtype=torch.bool)
    untouched[X, Y] = False
    assert bool((got[untouched] == 1.0).all()), "pixels without a vertex keep the canvas colour"


# ---- the exact CUDA-core kernel (query_fp32.cu): default path of the colour head, fallback for every other head shape ----
@pytest.fixture(scope="module")
def emu_query_fp32(tmp_path_factory):
    return build(tmp_path_factory, "emu_query_fp32")


@pytest.mark.parametrize("name,n", [("c_rot33", 200), ("c_identity", 100), ("g_persp", 150), ("g_nocalib", 77), ("g_identity", 130)])
def test_fp32_kernel_matches_reference_golden(emu_query_fp32, tmp_path, name, n):
    import torch
    from helpers import load_query_case
    case = load_query_case(name)
    res = case["expected"].shape[0]
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.f32")
    write_input(fin, case["feat"], case["points"][:, :, :n], case["calib"], case["proj"], res, case["last_op"], case["Ws"],
                case["bs"])
    r = subprocess.run([emu_query_fp32, fin, fout], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    got = torch.from_numpy(np.fromfile(fout, dtype=np.float32)).reshape(res, n)
    want = case["expected"][:, :n]
    assert (got - want).abs().max().item() <= 2e-5          # the GPU bar of the fp32 mode
    assert torch.equal(got[want == 0], want[want == 0]), "out-of-image points must be exactly 0"
