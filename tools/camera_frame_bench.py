"""What a per-frame camera costs in the captured frame.  The demo's default view mode (AUTO) turns the camera every frame
(yaw 20 deg, pitch +3 deg per frame through pifu_calib); FrameGraph.launch(x, calib=...) writes each frame's camera into the
graph's device buffer before the replay.  Arms, on bench.py's synthetic person (257^3 Seg3dLossless, faster=True, features
given) and a seeded netC head on a 512-channel map:
  - the eager chain with the frame's camera: geometry only (engine + forward_vertices), and the whole frame (+ the analytic
    normal image and the netC colour image);
  - FrameGraphRing at 1, 2 and 4 lanes with the AUTO camera per frame, geometry only and whole frame;
  - the same rings with a fixed camera (launch without a calib).

    python tools/camera_frame_bench.py [--rounds 3] [--window 1.0]

Outputs are compared before anything is timed: every ring's frames equal the eager chain's with the same camera, bit for
bit.  Every arm is warmed up, then timed in synchronised windows of at least `--window` seconds, the arms alternating round
after round; the line of an arm gives the range over the rounds.  The card's name and power limit are printed from the same
run."""
import argparse
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--window", type=float, default=1.0)
    args = ap.parse_args()
    import numpy as np
    import torch
    import bench
    from oracle import spec
    from monoport_b200.engine import Seg3dLossless, make_query_func
    from monoport_b200.modeling import PIFuNetC, PIFuNetG
    from monoport_b200.pipeline import FrameGraph, FrameGraphRing
    from monoport_b200.recon import colorization, forward_vertices, surface_normals

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    print("card: %s, power limit: %s" % (torch.cuda.get_device_name(dev), power))

    _, Ws, bs, feats_cpu = bench.synthetic(n_feat=4)
    torch.manual_seed(0)
    net = PIFuNetG()
    net.surface_classifier.load_state_dict({**{"filters.%d.weight" % l: W[:, :, None] for l, W in enumerate(Ws)},
                                            **{"filters.%d.bias" % l: b for l, b in enumerate(bs)}})
    net.surface_classifier.to(dev)
    net.eval()
    netC = PIFuNetC()
    netC.to(dev)
    netC.eval()
    feats = [f.to(dev) for f in feats_cpu]
    gC = torch.Generator().manual_seed(11)
    featsC = [(torch.randn(1, 512, 128, 128, generator=gC) * 0.5).to(dev) for _ in range(4)]
    b = np.array([bench.B_MIN], dtype=np.float32)
    eng = Seg3dLossless(make_query_func(net), b, -b, [17, 33, 65, 129, 257], balance_value=0.5, faster=True).to(dev)
    R = 257
    b_min, b_max = b[0], -b[0]
    # the demo's AUTO sequence (RTL/main.py update_camera: pitch + 3 deg per frame), 120 frames = one turn
    cams = [spec.scene_calib(20, 3 * k) for k in range(120)]
    cams_dev = [c.to(dev) for c in cams]
    fixed = cams[0]

    @torch.no_grad()
    def eager_frame(i, whole):
        cal = cams_dev[i % len(cams)]
        sdf = eng(im_feat_list=[[feats[i % 4]]], calib_tensor=cal)
        if sdf is None:
            return None
        X, Y, Z, N = forward_vertices(sdf, "front")
        if not whole:
            return sdf, X, Y, Z, N
        Ng = surface_normals(net, [[feats[i % 4]]], X, Y, Z, cal, R, b_min, b_max, precision="auto")
        rnorm = colorization(netC, None, X, Y, Z, cal, norm=Ng, resolution=R)
        rtex = colorization(netC, [[featsC[i % 4]]], X, Y, Z, cal, resolution=R)
        return sdf, X, Y, Z, N, rnorm, rtex

    def geo(n):
        return (feats[i % 4] for i in range(n))

    def whole(n):
        return ((feats[i % 4], featsC[i % 4]) for i in range(n))

    def per_frame(n):
        return [cams[i % len(cams)] for i in range(n)]

    rings = {}
    for lanes in (1, 2, 4):
        rings["graph geometry only, %d lane(s)" % lanes] = (FrameGraphRing(
            lambda: FrameGraph(net, eng, fixed, "front", with_encoder=False), n_lanes=lanes), geo)
        rings["graph whole frame, %d lane(s)" % lanes] = (FrameGraphRing(
            lambda: FrameGraph(net, eng, fixed, "front", with_encoder=False, netC=netC, render_normals="gradient"),
            n_lanes=lanes), whole)

    # ---- the outputs first: every ring's frames equal the eager chain with the same camera
    for lanes in (1, 2, 4):
        for kind, is_whole in (("geometry only", False), ("whole frame", True)):
            ring, gen = rings["graph %s, %d lane(s)" % (kind, lanes)]
            for i, out in enumerate(ring.run(gen(6), calibs=per_frame(6))):
                w = eager_frame(i, is_whole)
                for a, g in zip(w, out):
                    assert a.shape == g.shape and torch.equal(a, g), "%s, %d lanes: frame %d differs" % (kind, lanes, i)
    print("outputs checked: every ring frame equals the eager chain with its camera")

    # ---- timing: warm-up, then alternating windows of at least args.window seconds
    def eager_variant(is_whole):
        def run(n):
            for i in range(n):
                eager_frame(i, is_whole)
        return run

    def ring_variant(ring, gen, moving):
        def run(n):
            for _ in ring.run(gen(n), calibs=per_frame(n) if moving else None):
                pass
        return run

    variants = {"eager chain, geometry only (AUTO camera)": eager_variant(False),
                "eager chain, whole frame (AUTO camera)": eager_variant(True)}
    for name, (ring, gen) in rings.items():
        variants[name + ", AUTO camera"] = ring_variant(ring, gen, True)
        variants[name + ", fixed camera"] = ring_variant(ring, gen, False)
    for run in variants.values():
        run(8)
    torch.cuda.synchronize()
    rates = {k: [] for k in variants}
    for _ in range(args.rounds):
        for name, run in variants.items():
            n, t = 8, 0.0
            while True:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                run(n)
                torch.cuda.synchronize()
                t = time.perf_counter() - t0
                if t >= args.window:
                    break
                n = int(n * max(2.0, 1.2 * args.window / max(t, 1e-3)))
            rates[name].append(n / t)
    for name, r in rates.items():
        print("%-58s %8.1f - %8.1f frames/s" % (name, min(r), max(r)))
    for ring, _ in rings.values():
        ring.close()


if __name__ == "__main__":
    main()
