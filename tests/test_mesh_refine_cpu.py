"""CPU checks of the mesh refinement (mp_mesh_refine_async, DESIGN.md §F3.1): mesh_edges_kernel, refine_init_kernel and
refine_step_kernel run unmodified on the CPU model (tests/emu/emu_mesh_refine.cpp) after marching cubes, with every grid
forced to 1-3 CTAs.  The edge records must reproduce the emitted vertices bit for bit, the update must be the float32
restatement's (tests/mesh_refine_ref.py) bit for bit for given values per round, and the new kernels compile without a stack
frame while the marching-cubes kernels keep their machine code.  The restatement itself is checked against the accuracy
bars of the GPU tests on a small person volume."""
import hashlib
import re
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from emu_harness import EMU, HAVE_GXX, ptxas_report
from mesh_refine_ref import edge_world_points, mc_edges, query64, refine_mesh_ref, world_scale
from oracle import spec


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    """tests/emu/emu_mesh_refine.cpp, compiled once per module with the recipe of emu_harness.build for the integer / byte
    harnesses (-O1, no CUDA headers, no FP contraction)"""
    if not HAVE_GXX:
        pytest.skip("g++ not available")
    exe = tmp_path_factory.mktemp("emu_mesh_refine") / "emu_mesh_refine"
    cmd = ["g++", "-std=c++17", "-O1", "-march=native", "-pthread", "-ffp-contract=off", "-Wno-unknown-pragmas",
           "-fno-strict-aliasing", "-DMP_CUDA_EMU=1", "-I" + EMU, "-o", str(exe), EMU + "/emu_mesh_refine.cpp"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return str(exe)


def _run(exe, tmp_path, vol, v_cap, blocks, eager=0, world=1, b_min=(-1, -1, -1), b_max=(1, 1, 1), sigma=None, rounds=0,
         iso=0.5):
    D, H, W = vol.shape
    np.ascontiguousarray(vol, dtype=np.float32).tofile(tmp_path / "vol.f32")
    sig = np.zeros(0, np.float32) if sigma is None else np.ascontiguousarray(sigma, dtype=np.float32)
    sig.tofile(tmp_path / "sigma.f32")
    argv = [exe, D, H, W, repr(float(np.float32(iso))), v_cap, blocks, eager, world, W, *b_min, *b_max, rounds,
            tmp_path / "vol.f32", tmp_path / "sigma.f32", tmp_path]
    r = subprocess.run([str(a) for a in argv], capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stderr[-2000:]
    nv, nf, c32 = (int(x) for x in r.stdout.split())
    kv = min(nv, v_cap)
    out = dict(nv=nv, nf=nf, count32=c32,
               verts_mc=np.fromfile(tmp_path / "verts_mc.f32", np.float32).reshape(kv, 3),
               node=np.fromfile(tmp_path / "edge_node.u32", np.uint32),
               axis=np.fromfile(tmp_path / "edge_axis.u8", np.uint8))
    if not eager:
        out["rows"] = np.fromfile(tmp_path / "rows.f32", np.float32).reshape(rounds, 3, c32)
        out["verts"] = np.fromfile(tmp_path / "verts.f32", np.float32).reshape(c32, 3)
    return out


def _t0_points(vol, node, axis, world, b_min, b_max, iso=0.5):
    """the point at t0 on each recorded edge, with the emission's roundings (index space, or world)"""
    D, H, W = vol.shape
    node = node.astype(np.int64)
    zz, rem = node // (H * W), node % (H * W)
    yy, xx = rem // W, rem % W
    aa = axis.astype(np.int64)
    flat = np.ascontiguousarray(vol, dtype=np.float32).reshape(-1)
    step = np.where(aa == 0, 1, np.where(aa == 1, W, H * W))
    va, vb = torch.from_numpy(flat[node]), torch.from_numpy(flat[node + step])
    t0 = (torch.tensor(np.float32(iso)) - va) / (vb - va)
    if world:
        return edge_world_points(xx, yy, zz, aa, t0, *world_scale(W, b_min, b_max)).numpy()
    p = torch.from_numpy(np.stack([xx, yy, zz], 1)).to(torch.float32)
    p[torch.arange(len(aa)), torch.from_numpy(aa)] += t0
    return p.numpy()


def _same_bits(a, b):
    return a.shape == b.shape and np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))


KINDS = ["sphere", "corner", "slab", "ball01", "steps", "two_blobs", "noise"]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("mode", ["index", "world", "eager"])
@pytest.mark.parametrize("blocks", [1, 3])
def test_edge_records_reproduce_the_emitted_vertices(emu, tmp_path, kind, mode, blocks):
    """every emitted vertex's (node, axis) record gives its t0 point bit for bit, in spec.marching_cubes_ref's edge order"""
    R = 13 if kind == "noise" else 17
    vol = spec.analytic_volume(R, kind)
    b_min, b_max = (-1.0, -0.75, -1.25), (1.0, 1.25, 0.5)
    out = _run(emu, tmp_path, vol, 3 * R ** 3, blocks, eager=int(mode == "eager"), world=int(mode == "world"), b_min=b_min,
               b_max=b_max)
    nv = out["nv"]
    assert nv > 0 and out["node"].shape == (nv,)
    xx, yy, zz, aa = mc_edges(vol)
    assert np.array_equal(out["node"], (zz * R * R + yy * R + xx).astype(np.uint32)) and np.array_equal(out["axis"], aa)
    pts = _t0_points(vol, out["node"], out["axis"], mode == "world", b_min, b_max)
    assert _same_bits(pts, out["verts_mc"]), mode
    if mode != "world":
        assert _same_bits(out["verts_mc"], spec.marching_cubes_ref(vol)[0])


@pytest.mark.parametrize("blocks", [1, 2])
def test_no_record_at_or_beyond_the_capacity(emu, tmp_path, blocks):
    vol = spec.analytic_volume(17, "two_blobs")
    full = _run(emu, tmp_path, vol, 8 * 17 * 17, blocks)
    for v_cap in (full["nv"] - 5, 1, 0):
        out = _run(emu, tmp_path, vol, v_cap, blocks)           # (the harness checks the guard words itself)
        assert out["nv"] == full["nv"] and out["count32"] == v_cap
        assert np.array_equal(out["node"], full["node"][:v_cap]) and np.array_equal(out["axis"], full["axis"][:v_cap])


def _field(p):
    """a smooth value field near the sphere of analytic_volume, unclipped: sigma = 0.5 + 4 (0.6 - |p| + 0.02 sin(7x))"""
    p = p.double()
    d = p.norm(dim=0)
    return (0.5 + 4.0 * (0.6 - d + 0.02 * torch.sin(7.0 * p[0]))).float()


def _scripted(special):
    """query_fn of the restatement: _field, with the cases of `special` (vertex ids -> rule) applied, recording each
    round's values for the harness"""
    rec = []

    def fn(p):
        s = _field(p)
        n = s.shape[0]
        r = len(rec)
        ids = torch.arange(n)
        s = torch.where(ids % 7 == 0, torch.zeros_like(s), s)                # outside the image: sigma = 0
        s = torch.where(ids % 11 == 3, 1.0 - s, s)                           # the network's sign disagrees with the volume's
        if "zero" in special:
            s = torch.where((ids % 5 == 1) & (r == 1), torch.full_like(s, 0.5), s)   # a root hit exactly in round 1
        if "ties" in special:
            s = torch.where(ids % 13 == 2, torch.full_like(s, 0.75), s)      # the same |f| every round
        rec.append(s.clone())
        return s
    return fn, rec


@pytest.mark.parametrize("rounds", [0, 1, 2, 8])
@pytest.mark.parametrize("special", ["zero", "ties"])
@pytest.mark.parametrize("blocks", [1, 3])
def test_update_matches_the_restatement(emu, tmp_path, rounds, special, blocks):
    """the query rows of every round and the written vertices equal refine_mesh_ref's bit for bit"""
    vol = spec.analytic_volume(17, "sphere")
    b_min, b_max = (-1.0, -1.0, -1.0), (1.0, 1.0, 1.0)
    fn, rec = _scripted(special)
    want, _, rows = refine_mesh_ref(fn, vol, 0.5, rounds, b_min, b_max, trace=True)
    # (the last round's values come from the restatement's final query; earlier rounds' equal its recorded ones)
    sigma = torch.stack(rec).numpy() if rounds else np.zeros((0,), np.float32)
    out = _run(emu, tmp_path, vol, 8 * 17 * 17, blocks, sigma=sigma, rounds=rounds, b_min=b_min, b_max=b_max)
    assert out["count32"] == out["nv"] == want.shape[0]
    for r in range(rounds):
        assert _same_bits(out["rows"][r], rows[r].t().contiguous().numpy()), r
    assert _same_bits(out["verts"], want.numpy())
    if rounds <= 1:
        assert _same_bits(out["verts"], out["verts_mc"])
    # on the edge: the two other coordinates keep the marching-cubes vertex's bits
    mc, got = torch.from_numpy(out["verts_mc"]), torch.from_numpy(out["verts"])
    _, _, _, aa = mc_edges(vol)
    keep = torch.ones_like(mc, dtype=torch.bool)
    keep[torch.arange(len(aa)), torch.as_tensor(aa)] = False
    assert torch.equal(got[keep], mc[keep])


def test_capacity_below_the_vertex_count_refines_the_prefix(emu, tmp_path):
    vol = spec.analytic_volume(17, "sphere")
    fn, rec = _scripted("zero")
    want, _ = refine_mesh_ref(fn, vol, 0.5, 3, (-1, -1, -1), (1, 1, 1))
    full = torch.stack(rec).numpy()
    v_cap = want.shape[0] - 37
    out = _run(emu, tmp_path, vol, v_cap, 2, sigma=np.ascontiguousarray(full[:, :v_cap]), rounds=3)
    assert out["count32"] == v_cap
    assert _same_bits(out["verts"], want[:v_cap].numpy())


def test_empty_volume(emu, tmp_path):
    out = _run(emu, tmp_path, np.zeros((9, 9, 9), np.float32), 64, 2, sigma=np.zeros(0, np.float32), rounds=4)
    assert out["nv"] == 0 and out["verts"].shape == (0, 3)


# ---- compiler
NEW_KERNELS = ("mesh_edges_kernel", "refine_init_kernel", "refine_step_kernel")


def test_new_kernels_have_no_stack_frame_and_no_spills():
    entries, _ = ptxas_report("mcubes.cu")
    seen = set()
    for name, lines in entries:
        k = next((k for k in NEW_KERNELS if k in name), None)
        if k is None:
            continue
        seen.add(k)
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", " ".join(lines))
        assert m and m.groups() == ("0", "0", "0"), (name, lines)
    assert seen == set(NEW_KERNELS)


# sha-256 (first 16 hex digits) of the instructions and encodings of the marching-cubes kernels, compiled by nvcc 12.9 with the
# library's flags: the refinement shares their vertex arithmetic through inline helpers and must not change their code
MC_SASS = {
    "_ZN6mcubes11bits_kernelEPKfPjxf": "91d24728c00e395f",
    "_ZN6mcubes20classify_sums_kernelEPKjPNS_8WordInfoExiiiPyiS4_": "af05d31f42ad7166",
    "_ZN6mcubes16mesh_emit_kernelEPKfPKjPKNS_8WordInfoEPKyS3_jPfPiiiixf": "4bdd7b0b624a9653",
    "_ZN6mcubes22mesh_emit_async_kernelEPKfPKjPKNS_8WordInfoEPKyS3_S3_S8_NS_7MeshOutEPxPiiiixf": "d3a21460c534a5dc",
}


def _sass_hashes(sass):
    out, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            out[cur] = []
            continue
        if cur is None:
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4}\*/\s*(.*?)\s*;?\s*/\* (0x[0-9a-f]+) \*/", line)
        if m:
            out[cur].append(m.group(1) + " " + m.group(2))
            continue
        m = re.match(r"\s*/\* (0x[0-9a-f]+) \*/", line)
        if m:
            out[cur].append(m.group(1))
    return {k: hashlib.sha256("\n".join(v).encode()).hexdigest()[:16] for k, v in out.items()}


def test_marching_cubes_kernels_keep_their_machine_code():
    from monoport_b200 import build as lib_build
    try:
        nvcc = lib_build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not available")
    ver = subprocess.run([nvcc, "--version"], capture_output=True, text=True).stdout
    if "release 12.9" not in ver:
        pytest.skip("the pinned machine code is nvcc 12.9's")
    cuobjdump = nvcc[:-len("nvcc")] + "cuobjdump"
    with tempfile.TemporaryDirectory() as d:
        obj = d + "/mcubes.o"
        r = subprocess.run([nvcc] + lib_build.NVCC_FLAGS + ["-c", lib_build.CSRC + "/mcubes.cu", "-o", obj], capture_output=True,
                           text=True)
        assert r.returncode == 0, r.stderr[-2000:]
        sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    got = _sass_hashes(sass)
    for name, h in MC_SASS.items():
        assert got.get(name) == h, name


# ---- the accuracy bars of the GPU tests, on the restatement
def test_restatement_meets_the_accuracy_bar_on_a_person_volume():
    """fp32 spec.query_ref as the network, K = 8, at R = 33: over vertices whose float64 end values bracket iso, the p99 of
    |sigma64(v) - iso| is <= 1e-4 (the bar of the GPU test in "fp32"); the marching-cubes vertices' figure is printed beside it"""
    torch.manual_seed(0)
    Ws, bs = spec.make_weights(spec.G_CHANNELS, 3)
    Ws, bs, feat, _ = spec.heightfield_person(Ws, bs, spec.make_feat(256, 64, 64, 4, 0.5))
    cal = spec.scene_calib(20, 33)
    R, b_min, b_max = 33, (-1.0, -1.0, -1.0), (1.0, 1.0, 1.0)
    r = (torch.arange(R, dtype=torch.float32) + 0.5) / R * 2 - 1
    z, y, x = torch.meshgrid(r, r, r, indexing="ij")
    grid = torch.stack([x.reshape(-1), y.reshape(-1), z.reshape(-1)])
    vol = spec.query_ref(feat, grid, cal, Ws, bs, spec.LAST_SIGMOID)[0].reshape(R, R, R).numpy()

    def q32(p):
        return spec.query_ref(feat, p, cal, Ws, bs, spec.LAST_SIGMOID)[0]

    def q64(p):
        return query64(feat, p, cal, Ws, bs)[0]
    mc, _ = refine_mesh_ref(q32, vol, 0.5, 0, b_min, b_max)
    ref, _ = refine_mesh_ref(q32, vol, 0.5, 8, b_min, b_max)
    xx, yy, zz, aa = mc_edges(vol)
    lo, sc = torch.tensor(b_min, dtype=torch.float64), torch.tensor(b_max, dtype=torch.float64) - torch.tensor(b_min, dtype=torch.float64)
    base = torch.stack([torch.as_tensor(xx), torch.as_tensor(yy), torch.as_tensor(zz)], 1).double()
    ends = []
    for k in (0, 1):
        p = base.clone()
        p[torch.arange(len(aa)), torch.as_tensor(aa)] += k
        ends.append(q64(((p + 0.5) * sc / R + lo).t()) - 0.5)
    bracket = (ends[0] > 0) != (ends[1] > 0)
    e_mc = (q64(mc.t().double()) - 0.5).abs()[bracket]
    e_ref = (q64(ref.t().double()) - 0.5).abs()[bracket]
    p99 = lambda e: torch.quantile(e, 0.99).item()
    print("R=33, %d of %d vertices bracketed: |sigma64 - iso| p99 MC %.3e, refined (K=8) %.3e; max %.3e / %.3e"
          % (int(bracket.sum()), len(aa), p99(e_mc), p99(e_ref), e_mc.max().item(), e_ref.max().item()))
    assert int(bracket.sum()) > 0.9 * len(aa)
    assert p99(e_ref) <= 1e-4 and p99(e_ref) < p99(e_mc)
