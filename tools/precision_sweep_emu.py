"""Precision sweep of the tensor-core programs on the CPU model of the wgmma layer (no GPU needed):
max / mean |kernel - oracle| of query() outputs over seeded heads x feature maps x calibrations.
Usage: python tools/precision_sweep_emu.py [n_seeds] [n_points] [map_size]   (builds tests/emu/emu_query_tc.cpp into /tmp)"""
import os, struct, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np, torch
from oracle import spec

S = int(sys.argv[1]) if len(sys.argv) > 1 else 8
N = int(sys.argv[2]) if len(sys.argv) > 2 else 512
HW = int(sys.argv[3]) if len(sys.argv) > 3 else 32
exe = "/tmp/emu_query_tc_sweep"
emu = os.path.join(ROOT, "tests", "emu")
subprocess.run(["g++", "-std=c++17", "-O2", "-pthread", "-ffp-contract=off", "-fno-strict-aliasing", "-DMP_CUDA_EMU=1",
                "-I/usr/local/cuda/include", "-I" + emu, "-Wno-unknown-pragmas", "-o", exe, os.path.join(emu, "emu_query_tc.cpp")], check=True)
for net, chans, last in (("G", spec.G_CHANNELS, spec.LAST_SIGMOID), ("C", spec.C_CHANNELS, spec.LAST_TANH)):
    for prog in ((2, 3) if net == "G" else (0,)):
        worst, mean = 0.0, 0.0
        for s in range(S):
            Ws, bs = spec.make_weights(chans, 1000 + s)
            feat = spec.make_feat(chans[0] - 1, HW, HW, 2000 + s)
            pts = spec.make_points(N, 3000 + s)
            cal = spec.scene_calib(20, -60 + 17 * s)
            want = spec.query_ref(feat, pts, cal, Ws, bs, last)
            with open("/tmp/sweep_in.bin", "wb") as f:
                f.write(struct.pack("8i", chans[0] - 1, HW, HW, N, 1, 0, chans[-1], last))
                f.write(struct.pack("f", spec.Z_SCALE))
                f.write(struct.pack("12f", *cal[0, :3, :4].reshape(-1).tolist()))
                f.write(feat.numpy().tobytes()); f.write(pts[0].numpy().tobytes())
                for W, b in zip(Ws, bs):
                    f.write(W.numpy().tobytes()); f.write(b.numpy().tobytes())
            r = subprocess.run([exe, "/tmp/sweep_in.bin", "/tmp/sweep_out.f32", str(prog), "4"], capture_output=True, text=True)
            assert r.returncode == 0, r.stderr
            got = torch.from_numpy(np.fromfile("/tmp/sweep_out.f32", dtype=np.float32)).reshape(chans[-1], N)
            e = (got - want).abs()
            worst, mean = max(worst, e.max().item()), mean + e.mean().item() / S
        name = {2: "geometry head, program v2", 3: "geometry head, program v3", 0: "colour head (query_tc3c_kernel)"}[prog]
        print("%-34s max |kernel - oracle| = %.3e   mean = %.3e   (%d seeds x %d points, %dx%d map)" % (name, worst, mean, S, N, HW, HW))
