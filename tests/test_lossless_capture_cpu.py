"""CPU checks of the device-driven conflict loop of the lossless engine (mp_octree_run_fused_async): the engine's kernels,
loop_control_kernel included, run unmodified on the CPU model (tests/emu/emu_octree_loop.cpp) with the loop-control kernel
deciding whether another pass runs, as the WHILE node's condition does on the GPU.  Volume, node lists and per-level counts
must equal the restatement's, and the passes per level its query calls per level.  A cap below the walk's length stops the
level and sets the truncated flag.  Also: loop_control_kernel compiles for sm_90a without a stack frame or spills."""
import re
import subprocess

import numpy as np
import pytest
import torch

from oracle import spec
from emu_harness import build, ptxas_report
from helpers import lookup_query


def rod_field(R):
    """The sphere of analytic_volume plus a one-voxel-wide diagonal rod leaving it: a thin feature the coarse levels miss,
    which the conflict loop has to walk node by node."""
    f = spec.analytic_volume(R, "sphere")
    c = R // 2
    for t in range(R // 2):
        f[c + 1, c + t, c + t] = 1.0
        f[c + 1, c + t, c + t + 1] = 1.0
    return f


@pytest.fixture(scope="module")
def emu_octree(tmp_path_factory):
    return build(tmp_path_factory, "emu_octree_loop")


def _run_loop(exe, tmp_path, field, res, cap=0):
    fin, fvol, fidx = (str(tmp_path / n) for n in ("dense.f32", "vol.f32", "idx.i32"))
    np.ascontiguousarray(field, dtype=np.float32).tofile(fin)
    args = [exe, "0.5", fin, fvol, fidx, str(cap), str(len(res))] + [str(r) for r in res]
    r = subprocess.run(args, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr
    first, second = r.stdout.strip().split("\n")
    out = [int(x) for x in first.split()]
    loops = [int(x) for x in second.split()]
    return out[0], out[1:], loops[:-1], loops[-1], np.fromfile(fvol, dtype=np.float32), np.fromfile(fidx, dtype=np.int32)


def _oracle(field, res):
    """The restatement's volume, per-level node lists and number of query calls per level."""
    fn_o, _ = lookup_query(torch.from_numpy(field))
    sizes = []

    def fn(p):
        sizes.append(int(p.shape[0]))
        return fn_o(p)
    want, stats = spec.seg3d_lossless_ref(fn, res, faster=False, return_stats=True)
    # the calls come level after level and every call has points: split them by the per-level totals
    calls, k = [], 0
    for s in stats:
        total, n = int(s["idx"].numel()), 0
        while total > 0:
            total -= sizes[k]
            k += 1
            n += 1
        assert total == 0
        calls.append(n)
    assert k == len(sizes)
    return want, stats, calls


@pytest.mark.parametrize("kind,res", [("sphere", [9, 17]), ("ellipsoid", [9, 17, 33]), ("rod", [9, 17, 33])])
def test_device_loop_matches_restatement(emu_octree, tmp_path, kind, res):
    R = res[-1]
    field = rod_field(R) if kind == "rod" else spec.analytic_volume(R, kind)
    want, stats, calls = _oracle(field, res)
    nonempty, counts, passes, truncated, vol, idx = _run_loop(emu_octree, tmp_path, field, res)
    assert nonempty == 1 and want is not None and truncated == 0
    assert counts == [int(s["idx"].numel()) for s in stats]
    assert np.array_equal(vol.reshape(R, R, R), want.numpy()), "volume must be bit-identical to the restatement"
    assert np.array_equal(idx, np.concatenate([s["idx"].numpy().astype(np.int32) for s in stats])), "node lists / order"
    assert passes == [0] + [max(1, c) for c in calls[1:]], (passes, calls)
    if kind == "rod":
        assert passes[-1] == 9, passes           # the rod is walked one pass per node


def test_device_loop_stops_at_its_cap(emu_octree, tmp_path):
    field = rod_field(33)
    nonempty, counts, passes, truncated, vol, idx = _run_loop(emu_octree, tmp_path, field, [9, 17, 33], cap=3)
    assert nonempty == 1
    assert passes[-1] == 3 and truncated == 3, (passes, truncated)
    want, stats, _ = _oracle(field, [9, 17, 33])
    assert counts[-1] < int(stats[-1]["idx"].numel())


def test_loop_control_kernel_has_no_stack_frame():
    at = [lines for name, lines in ptxas_report("octree.cu")[0] if "loop_control_kernel" in name]
    assert len(at) == 1, "loop_control_kernel not compiled"
    stats = " ".join(at[0])
    m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", stats)
    assert m and m.groups() == ("0", "0", "0"), stats
