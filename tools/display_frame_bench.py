"""What the demo's display step costs beside the captured frame.  visulization (RTL/main.py:252-281) turns the two [R,R,3]
images into what the main loop shows: x255, rot90, nearest resize to 256 x 256, a host copy per image and the mask.  Arms,
on bench.py's synthetic person (257^3 Seg3dLossless, faster=True, features given) with a seeded netC head on a 512-channel
map and the normal image (render_normals=True), at 1 and 4 lanes:
  - FrameGraphRing with display=True: the display images made inside the captured step (mp_display_async);
  - the same ring without display, followed by the eager torch restatement visulization_ref (tests/display_cases.py) of
    every frame's rendered() images (what a program driving the demo with a ring had to run before);
  - the ring without display and without the eager step, as a reference point.

    python tools/display_frame_bench.py [--rounds 3] [--window 1.0]

Outputs are compared before anything is timed: every displayed() equals the restatement of its frame's images, bit for
bit.  Every arm is warmed up, then timed in synchronised windows of at least `--window` seconds, the arms alternating
round after round; the line of an arm gives the range over the rounds.  The card's name, power limit and SM clock are
printed from the same run."""
import argparse
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(1, os.path.join(ROOT, "tests"))         # display_cases: the torch restatement of visulization


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                               "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--window", type=float, default=1.0)
    args = ap.parse_args()
    import numpy as np
    import torch
    import bench
    from oracle import spec
    from display_cases import visulization_ref
    from monoport_b200.engine import Seg3dLossless, make_query_func
    from monoport_b200.modeling import PIFuNetC, PIFuNetG
    from monoport_b200.pipeline import FrameGraph, FrameGraphRing

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print("card (name, power limit, SM clock, max SM clock) before: %s" % _card())

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
    cal = spec.scene_calib(20, 0)

    def items(n):
        return ((feats[i % 4], featsC[i % 4]) for i in range(n))

    rings = {}
    for lanes in (1, 4):
        for display in (True, False):
            rings[(lanes, display)] = FrameGraphRing(
                lambda: FrameGraph(net, eng, cal, "front", with_encoder=False, netC=netC, render_normals=True,
                                   display=display), n_lanes=lanes)

    def same(a, b):                                       # bit for bit, NaN payloads included
        a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
        return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()

    # ---- the outputs first: the captured display images equal the restatement of the frame's images
    for lanes in (1, 4):
        for i, out in enumerate(rings[(lanes, True)].run(items(6))):
            shown, want = out[-3:], visulization_ref(out[5], out[6])
            assert all(same(a, w) for a, w in zip(shown, want)), "%d lanes: frame %d differs" % (lanes, i)
    print("outputs checked: every displayed() equals visulization_ref(*rendered()) bit for bit")

    def captured(ring):
        def run(n):
            for _ in ring.run(items(n)):
                pass
        return run

    def eager_tail(ring):
        def run(n):
            for out in ring.run(items(n)):
                visulization_ref(out[5], out[6])
        return run

    variants = {}
    for lanes in (1, 4):
        variants["captured display frame, %d lane(s)" % lanes] = captured(rings[(lanes, True)])
        variants["ring + eager visulization, %d lane(s)" % lanes] = eager_tail(rings[(lanes, False)])
        variants["captured frame without display, %d lane(s)" % lanes] = captured(rings[(lanes, False)])
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
    print("card (name, power limit, SM clock, max SM clock) after:  %s" % _card())
    for name, r in rates.items():
        print("%-48s %8.1f - %8.1f frames/s" % (name, min(r), max(r)))
    for ring in rings.values():
        ring.close()


if __name__ == "__main__":
    main()
