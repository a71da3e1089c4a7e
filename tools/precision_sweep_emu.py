"""Precision sweep of the tensor-core programs on the CPU model of the wgmma layer (no GPU needed):
max / mean |kernel - oracle| of query() outputs over seeded heads x feature maps x calibrations.
Usage: python tools/precision_sweep_emu.py [n_seeds] [n_points] [map_size]   (builds tests/emu/emu_tc.cpp into a temporary
directory)"""
import os, subprocess, sys, tempfile
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
from oracle import spec
from emu_harness import build, write_input

S = int(sys.argv[1]) if len(sys.argv) > 1 else 8
N = int(sys.argv[2]) if len(sys.argv) > 2 else 512
HW = int(sys.argv[3]) if len(sys.argv) > 3 else 32
with tempfile.TemporaryDirectory() as tmp:
    exe = build(tmp, "emu_tc")
    fin, fout = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.f32")
    for net, chans, last in (("geometry head", spec.G_CHANNELS, spec.LAST_SIGMOID),
                             ("colour head", spec.C_CHANNELS, spec.LAST_TANH)):
        worst, mean = 0.0, 0.0
        for s in range(S):
            Ws, bs = spec.make_weights(chans, 1000 + s)
            feat = spec.make_feat(chans[0] - 1, HW, HW, 2000 + s)
            pts = spec.make_points(N, 3000 + s)
            cal = spec.scene_calib(20, -60 + 17 * s)
            want = spec.query_ref(feat, pts, cal, Ws, bs, last)
            write_input(fin, feat, pts, cal, "orthogonal", chans[-1], last, Ws, bs)
            r = subprocess.run([exe, fin, fout, "query", "--sms", "4"], capture_output=True, text=True)
            assert r.returncode == 0, r.stderr
            got = torch.from_numpy(np.fromfile(fout, dtype=np.float32)).reshape(chans[-1], N)
            e = (got - want).abs()
            worst, mean = max(worst, e.max().item()), mean + e.mean().item() / S
        print("%-14s max |kernel - oracle| = %.3e   mean = %.3e   (%d seeds x %d points, %dx%d map)"
              % (net, worst, mean, S, N, HW, HW))
