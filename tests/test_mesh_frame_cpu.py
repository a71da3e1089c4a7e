"""CPU checks of the enqueue-only marching cubes (mp_mcubes_run_async): the kernels of mcubes_kernels.cuh run unmodified on
the CPU model (tests/emu/emu_mcubes_async.cpp) in the call's sequence, with the emission grid forced to 1-3 CTAs so that
every CTA walks several rounds of the active list.  The mesh must be the eager emission's (emu_mcubes) and the restatement's
(spec.marching_cubes_ref) bit for bit, in index space and in reconstruction()'s world space; the capacities must cut the
writes exactly while the true totals are still reported; two runs on one workspace must each equal a fresh run.  Also:
mesh_emit_async_kernel compiles for sm_90a without a stack frame or spills."""
import re
import subprocess

import numpy as np
import pytest
import torch

from oracle import spec
from emu_harness import build, needs_gxx, ptxas_report

pytestmark = needs_gxx


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return build(tmp_path_factory, "emu_mcubes_async"), build(tmp_path_factory, "emu_mcubes")


def _run_async(exe, vols, tmp_path, v_cap=None, f_cap=None, blocks=2, world=None, iso=0.5):
    """Runs the sequence once per volume on one workspace.  -> [(verts written, faces written, nV, nF, count32)]"""
    D, H, W = vols[0].shape
    ins = []
    for k, v in enumerate(vols):
        p = str(tmp_path / ("vol%d.f32" % k))
        np.ascontiguousarray(v, dtype=np.float32).tofile(p)
        ins.append(p)
    if world is None:
        wargs = ["0", "1", "0", "0", "0", "0", "0", "0"]
    else:
        R, lo, hi = world
        wargs = ["1", repr(float(R))] + [repr(float(x)) for x in lo] + [repr(float(x)) for x in hi]
    # default capacities: the largest mesh a volume of this shape can give (3 edges per node, 5 triangles per cell)
    vc = 3 * D * H * W if v_cap is None else v_cap
    fc = 5 * D * H * W if f_cap is None else f_cap
    args = [exe, str(D), str(H), str(W), repr(float(iso)), str(vc), str(fc), str(blocks)] + wargs + [str(tmp_path)] + ins
    r = subprocess.run(args, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr
    out = []
    for k, line in enumerate(r.stdout.strip().split("\n")):
        nv, nf, c32 = (int(x) for x in line.split())
        v = np.fromfile(str(tmp_path / ("verts%d.f32" % k)), dtype=np.float32).reshape(-1, 3)
        f = np.fromfile(str(tmp_path / ("faces%d.i32" % k)), dtype=np.int32).reshape(-1, 3)
        out.append((v, f, nv, nf, c32))
    return out


def _run_eager(exe, vol, tmp_path, iso=0.5):
    D, H, W = vol.shape
    vin, vout, fout = (str(tmp_path / n) for n in ("e_vol.f32", "e_verts.f32", "e_faces.i32"))
    np.ascontiguousarray(vol, dtype=np.float32).tofile(vin)
    r = subprocess.run([exe, str(D), str(H), str(W), repr(float(iso)), vin, vout, fout], capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr
    return np.fromfile(vout, dtype=np.float32).reshape(-1, 3), np.fromfile(fout, dtype=np.int32).reshape(-1, 3)


def _world_ref(V, R, b_min, b_max):
    """reconstruction()'s mapping, in torch: (v + 0.5) * ((b_max - b_min) / R) + b_min"""
    lo = torch.as_tensor(np.asarray(b_min, dtype=np.float32)).view(3)
    hi = torch.as_tensor(np.asarray(b_max, dtype=np.float32)).view(3)
    return ((torch.from_numpy(V) + 0.5) * ((hi - lo) / R) + lo).numpy()


@pytest.mark.parametrize("blocks", [1, 3])
@pytest.mark.parametrize("kind,R", [("sphere", 33), ("ellipsoid", 40), ("two_blobs", 49)])
def test_async_emission_matches_eager_and_oracle_on_analytic_volumes(emu, tmp_path, kind, R, blocks):
    exe, eager = emu
    vol = spec.analytic_volume(R, kind)
    V, F = spec.marching_cubes_ref(vol)
    ve, fe = _run_eager(eager, vol, tmp_path)
    (v, f, nv, nf, c32), = _run_async(exe, [vol], tmp_path, blocks=blocks)
    assert (nv, nf, c32) == (V.shape[0], F.shape[0], V.shape[0])
    assert np.array_equal(f, F) and np.array_equal(f, fe)
    assert np.array_equal(v, V) and np.array_equal(v, ve)


@pytest.mark.parametrize("shape", [(20, 17, 23), (9, 40, 35), (2, 2, 2), (3, 70, 2), (3, 5, 131), (2, 3, 257), (2, 9, 128),
                                   (2, 2, 33)])
def test_async_emission_matches_oracle_on_noise(emu, tmp_path, shape):
    exe, _ = emu
    vol = np.random.default_rng(sum(shape)).random(shape, dtype=np.float32)
    V, F = spec.marching_cubes_ref(vol)
    (v, f, nv, nf, _), = _run_async(exe, [vol], tmp_path, blocks=2)
    assert (nv, nf) == (V.shape[0], F.reshape(-1, 3).shape[0])
    assert np.array_equal(f, F.reshape(-1, 3))
    assert np.array_equal(v, V)


@pytest.mark.parametrize("b_min,b_max", [((-1.0, -1.0, -1.0), (1.0, 1.0, 1.0)), ((-0.37, -1.25, 0.1), (0.93, 0.8, 2.7))])
def test_world_space_vertices_equal_torch_mapping(emu, tmp_path, b_min, b_max):
    exe, _ = emu
    R = 33
    vol = spec.analytic_volume(R, "ellipsoid")
    V, F = spec.marching_cubes_ref(vol)
    (v, f, nv, nf, _), = _run_async(exe, [vol], tmp_path, world=(R, b_min, b_max))
    assert np.array_equal(f, F)
    want = _world_ref(V, R, b_min, b_max)
    assert v.dtype == want.dtype and np.array_equal(v, want), np.abs(v - want).max()


def test_capacity_cuts_the_writes_and_keeps_the_totals(emu, tmp_path):
    """Exact fit, one vertex short, one face short, zero: the buffers hold the first v_cap vertices / f_cap faces of the
    full mesh and nothing behind them (the harness checks its guard words); the totals are always the true ones."""
    exe, _ = emu
    vol = spec.analytic_volume(33, "sphere")
    V, F = spec.marching_cubes_ref(vol)
    nV, nF = V.shape[0], F.shape[0]
    for vc, fc in [(nV, nF), (nV - 1, nF), (nV, nF - 1), (0, 0), (0, nF), (nV, 0)]:
        (v, f, nv, nf, c32), = _run_async(exe, [vol], tmp_path, v_cap=vc, f_cap=fc, blocks=3)
        assert (nv, nf) == (nV, nF), (vc, fc)
        assert c32 == min(nV, vc)
        assert np.array_equal(v, V[:vc]) and np.array_equal(f, F[:fc]), (vc, fc)


@pytest.mark.parametrize("fill", [0.0, 1.0])
def test_empty_volume(emu, tmp_path, fill):
    exe, _ = emu
    (v, f, nv, nf, c32), = _run_async(exe, [np.full((9, 9, 9), fill, dtype=np.float32)], tmp_path)
    assert (nv, nf, c32) == (0, 0, 0) and v.shape[0] == 0 and f.shape[0] == 0


def test_replay_on_one_workspace(emu, tmp_path):
    """The replay case: a larger mesh, a smaller one, an empty volume and the first again on one workspace and one set of
    buffers -- every run equals a fresh run (the per-run words are reset inside the sequence)."""
    exe, _ = emu
    R = 33
    a = spec.analytic_volume(R, "sphere")
    b = spec.analytic_volume(R, "two_blobs")
    c = np.zeros((R, R, R), dtype=np.float32)
    runs = _run_async(exe, [a, b, c, a], tmp_path, blocks=2, world=(R, (-1, -1, -1), (1, 1, 1)))
    fresh = tmp_path / "fresh"
    fresh.mkdir()
    for vol, (v, f, nv, nf, c32) in zip([a, b, c, a], runs):
        (v0, f0, nv0, nf0, c0), = _run_async(exe, [vol], fresh, blocks=2, world=(R, (-1, -1, -1), (1, 1, 1)))
        assert (nv, nf, c32) == (nv0, nf0, c0)
        assert np.array_equal(v, v0) and np.array_equal(f, f0)
    assert runs[0][2] > runs[1][2] > 0 and runs[2][2] == 0


def test_async_emission_kernel_has_no_stack_frame():
    at = [lines for name, lines in ptxas_report("mcubes.cu")[0] if "mesh_emit_async_kernel" in name]
    assert len(at) == 1, "mesh_emit_async_kernel not compiled"
    stats = " ".join(at[0])
    m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", stats)
    assert m and m.groups() == ("0", "0", "0"), stats
