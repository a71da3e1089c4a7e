"""The mesh renderer (monoport_b200/csrc/raster_kernels.cuh, mp_render_mesh_async; DESIGN.md §F3.2) on the CPU model: its
three kernels, unmodified, equal the numpy restatement tests/raster_ref.py bit for bit on the cases of render_cases.py; the
restatement's own properties (one fragment per pixel on a tessellated plane, a hole-free silhouette of a closed mesh); and
the ptxas report of raster.cu."""
import subprocess

import numpy as np
import pytest
import scipy.ndimage

import raster_ref
import render_cases
from emu_harness import EMU, HAVE_GXX, ptxas_report

CASES = ["fv_sphere_33_ortho0", "fv_sphere_33_ortho33", "fv_two_blobs_65_ortho0", "fv_two_blobs_65_ortho33",
         "fv_corner_33_ortho0", "fv_corner_33_ortho33", "fv_noise_33_ortho0", "fv_noise_33_ortho33", "persp_near",
         "quad_large", "quad_guard", "quad_persp", "coincident", "degenerate", "beyond_count", "views3", "nonsquare_96x64"]


@pytest.fixture(scope="module")
def emu_raster(tmp_path_factory):
    """tests/emu/emu_raster.cpp, compiled once per module with the recipe of emu_harness.build for the integer / byte
    harnesses (-O1, no CUDA headers, no FP contraction)"""
    if not HAVE_GXX:
        pytest.skip("g++ not available")
    exe = tmp_path_factory.mktemp("emu_raster") / "emu_raster"
    cmd = ["g++", "-std=c++17", "-O1", "-march=native", "-pthread", "-ffp-contract=off", "-Wno-unknown-pragmas",
           "-fno-strict-aliasing", "-DMP_CUDA_EMU=1", "-I" + EMU, "-o", str(exe), EMU + "/emu_raster.cpp"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return str(exe)


@pytest.fixture(scope="module")
def all_cases(golden_dir):
    return render_cases.cases(golden_dir)


def run_emu(exe, tmp_path, c, normals=True, colours=True, setup_blocks=2, large_blocks=3):
    """the kernels on the CPU model -> (keys [V,H,W], normal or None, colour or None, large-face list length)"""
    V, W, H = c["mats"].shape[0], c["W"], c["H"]
    fin = tmp_path / "in.bin"
    with open(fin, "wb") as f:
        f.write(np.asarray(c["counts"], dtype=np.int64).tobytes())
        f.write(np.zeros(4, dtype=np.float32).tobytes())
        for key in ("mats", "verts", "faces"):
            f.write(np.ascontiguousarray(c[key]).tobytes())
        if normals:
            f.write(np.ascontiguousarray(c["normals"], dtype=np.float32).tobytes())
        if colours:
            f.write(np.ascontiguousarray(c["colours"], dtype=np.float32).tobytes())
    r = subprocess.run([exe, str(c["verts"].shape[0]), str(c["faces"].shape[0]), str(V), str(W), str(H), str(int(normals)),
                        str(int(colours)), str(setup_blocks), str(large_blocks), str(fin), str(tmp_path)],
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-2000:]
    keys = np.fromfile(tmp_path / "keys.u64", dtype=np.uint64).reshape(V, H, W)
    img = [np.fromfile(tmp_path / ("%s.f32" % n), dtype=np.float32).reshape(V, H, W, 4) if on else None
           for n, on in (("normal", normals), ("colour", colours))]
    return keys, img[0], img[1], int(r.stdout)


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("name", CASES)
def test_kernels_equal_the_restatement(emu_raster, tmp_path, all_cases, name):
    c = all_cases[name]
    keys, normal, colour, listed = run_emu(emu_raster, tmp_path, c)
    want_keys, _, want_listed = raster_ref.raster(c["verts"], c["faces"], c["counts"], c["mats"], c["W"], c["H"])
    assert np.array_equal(keys, want_keys)
    assert listed == want_listed
    want_n, want_c = raster_ref.render(c["verts"], c["faces"], c["counts"], c["mats"], c["W"], c["H"], c["normals"],
                                       c["colours"])
    assert same_bits(normal, want_n) and same_bits(colour, want_c)
    assert (keys != raster_ref.CLEAR_KEY).any() or name == "degenerate"


def test_cases_cover_what_they_claim(all_cases):
    """the large-face path, clipping, the coincident tie, NaN normals and skipped faces actually occur"""
    def run(name):
        c = all_cases[name]
        return c, raster_ref.raster(c["verts"], c["faces"], c["counts"], c["mats"], c["W"], c["H"])
    c, (keys, frags, listed) = run("quad_large")
    assert listed == 2 and (keys != raster_ref.CLEAR_KEY).all() and frags.max() == 1
    c, (keys, frags, listed) = run("persp_near")
    assert listed > 0
    clip = np.stack([raster_ref.transform(c["mats"][0], c["verts"])])[0]
    assert (clip[:, 3] < 0).any() and (clip[:, 2] < -clip[:, 3]).any()            # behind the eye, through the near plane
    c, (keys, _, _) = run("coincident")
    hit = keys[keys != raster_ref.CLEAR_KEY]
    assert hit.size and ((hit & np.uint64(0xFFFFFFFF)) == 0).all()
    n, col = raster_ref.render(c["verts"], c["faces"], c["counts"], c["mats"], c["W"], c["H"], c["normals"], c["colours"])
    assert np.array_equal(np.unique(col[0, ..., :3][keys[0, ::-1] != raster_ref.CLEAR_KEY], axis=0), [[0, 1, 0]])
    c = all_cases["degenerate"]
    n, _ = raster_ref.render(c["verts"], c["faces"], c["counts"], c["mats"], c["W"], c["H"], c["normals"], c["colours"])
    assert np.isnan(n).any()
    c, (keys, _, _) = run("beyond_count")
    full = raster_ref.raster(c["verts"], c["faces"], np.array([len(c["verts"]), len(c["faces"])]), c["mats"], c["W"], c["H"])[0]
    assert not np.array_equal(keys, full)


def test_clear_colour_and_one_attribute(emu_raster, tmp_path, all_cases):
    """an attribute that is absent is not computed; the clear colour fills uncovered pixels"""
    c = all_cases["fv_sphere_33_ortho33"]
    keys, normal, colour, _ = run_emu(emu_raster, tmp_path, c, normals=False)
    assert normal is None
    _, want = raster_ref.render(c["verts"], c["faces"], c["counts"], c["mats"], c["W"], c["H"], None, c["colours"])
    assert same_bits(colour, want)
    empty = ~(keys[0, ::-1] != raster_ref.CLEAR_KEY)
    assert empty.any() and (colour[0][empty] == 0).all()


@pytest.mark.parametrize("W,H,seed", [(64, 64, 0), (96, 64, 1), (37, 53, 2)])
def test_tessellated_plane_gets_one_fragment_per_pixel(W, H, seed):
    """the top-left rule: pixels on edges shared by two faces are drawn once, none twice and none dropped"""
    m = render_cases.plane_mesh(7, seed)
    mats = raster_ref.view_mats(render_cases.model(0, 0, (0.013, -0.007, -2)), render_cases.demo_ortho())
    _, frags, _ = raster_ref.raster(m["verts"], m["faces"], (len(m["verts"]), len(m["faces"])), mats, W, H)
    assert frags.max() == 1
    # every pixel centre strictly inside the plane's square is covered
    i, j = np.meshgrid(np.arange(W), np.arange(H), indexing="xy")
    x, y = (2 * i + 1) / W - 1 - 0.013, (2 * j + 1) / H - 1 + 0.007
    inside = (np.abs(x) < 0.9 - 1e-3) & (np.abs(y) < 0.9 - 1e-3)
    assert (frags[0][inside] == 1).all()


@pytest.mark.parametrize("name,pitch,yaw", [("fv_sphere_33", 0, 0), ("fv_ellipsoid_65", 33, 20), ("fv_two_blobs_65", -15, 60)])
def test_closed_mesh_silhouette_has_no_holes(golden_dir, name, pitch, yaw):
    m = render_cases.golden_mesh(golden_dir, name)
    mats = raster_ref.view_mats(render_cases.model(pitch, yaw), render_cases.demo_ortho())
    keys, _, _ = raster_ref.raster(m["verts"], m["faces"], (len(m["verts"]), len(m["faces"])), mats, 128, 128)
    mask = keys[0] != raster_ref.CLEAR_KEY
    assert mask.sum() > 100
    assert np.array_equal(scipy.ndimage.binary_fill_holes(mask), mask)


def test_ptxas_report_has_no_spills():
    entries, _ = ptxas_report("raster.cu")
    names = [n for n, _ in entries]
    for k in ("raster_setup_kernel", "raster_large_kernel", "raster_resolve_kernel"):
        assert any(k in n for n in names), names
    for name, lines in entries:
        report = " ".join(lines)
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in report, (name, lines)
