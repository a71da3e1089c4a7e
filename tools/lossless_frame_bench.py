"""What the lossless coarse-to-fine engine (Seg3dLossless(faster=False)) costs per frame, eager against the captured frame
step (pipeline.FrameGraph, whose conflict loops run as conditional WHILE nodes decided on the device), with the captured
`faster` frame beside them.  Workload: bench.py's synthetic person, 257^3, features given, + forward_vertices.

    python tools/lossless_frame_bench.py [--rounds 3] [--window 1.0]

Variants:
  eager lossless                     engine(...) (mp_octree_run_fused: the host reads the list length after every pass)
                                     + forward_vertices
  eager lossless, device loop        mp_octree_run_fused_async on a stream that is not being captured (the call records
                                     its sequence into a graph, instantiates and launches it) + mp_octree_fetch +
                                     forward_vertices: what the device-driven loop costs an eager caller
  graph lossless, 1 / 2 lane(s)      FrameGraphRing over lossless frames
  graph faster, 1 / 2 lane(s)        FrameGraphRing over faster=True frames

The captured and eager lossless outputs are compared bit for bit before anything is timed.  Every variant is warmed up,
then timed in synchronised windows of at least `--window` seconds, the variants alternating round after round; the line
of a variant gives the range over the rounds.  The card's name and power limit are printed from the same run."""
import argparse
import ctypes
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
    from monoport_b200 import _lib
    from monoport_b200.engine import Seg3dLossless, make_query_func
    from monoport_b200.modeling import PIFuNetG
    from monoport_b200.pipeline import FrameGraph, FrameGraphRing
    from monoport_b200.recon import forward_vertices

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    print("card: %s, power limit: %s" % (torch.cuda.get_device_name(dev), power))

    _, Ws, bs, feats_cpu = bench.synthetic(n_feat=4)
    net = PIFuNetG()
    net.surface_classifier.load_state_dict({**{"filters.%d.weight" % l: W[:, :, None] for l, W in enumerate(Ws)},
                                            **{"filters.%d.bias" % l: b for l, b in enumerate(bs)}})
    net.surface_classifier.to(dev)
    net.eval()
    feats = [f.to(dev) for f in feats_cpu]
    cal = bench.scene_calib()
    calg = cal.to(dev)
    b = np.array([bench.B_MIN], dtype=np.float32)
    res = [17, 33, 65, 129, 257]
    R = res[-1]
    lossless = Seg3dLossless(make_query_func(net), b, -b, res, balance_value=0.5, faster=False).to(dev)
    faster = Seg3dLossless(make_query_func(net), b, -b, res, balance_value=0.5, faster=True).to(dev)

    def eager_frame(i):
        sdf = lossless(im_feat_list=[[feats[i % 4]]], calib_tensor=cal)
        X, Y, Z, N = forward_vertices(sdf, "front")
        return sdf, X, Y, Z, N

    # the device-driven loop for an eager caller: one handle, one output volume
    lib = _lib.load()
    h = lossless._new_handle(dev)
    vol = torch.empty((1, 1, R, R, R), dtype=torch.float32, device=dev)
    fh = net.feature_handle(feats[0])
    cal12 = _lib.calib12(cal)
    n_lv = len(res)

    @torch.no_grad()
    def eager_async_frame(i):
        f = feats[i % 4]
        fh.key = None
        fh.upload(f)
        st = _lib.stream_ptr(dev)
        _lib.check(lib.mp_octree_run_fused_async(h, net.surface_classifier.handle(), fh.ptr, cal12, _lib.PROJ_ORTHOGONAL,
                                                 ctypes.c_float(net.normalizer.scale), net._mode(),
                                                 ctypes.c_void_p(vol.data_ptr()), st), "mp_octree_run_fused_async")
        nonempty = ctypes.c_int(0)
        _lib.check(lib.mp_octree_fetch(h, ctypes.byref(nonempty), None, st), "mp_octree_fetch")
        if not nonempty.value:
            return None, None, None, None, None
        X, Y, Z, N = forward_vertices(vol, "front")
        return vol, X, Y, Z, N

    rings = {}
    for lanes in (1, 2):
        rings["graph lossless, %d lane(s)" % lanes] = FrameGraphRing(
            lambda: FrameGraph(net, lossless, cal, "front", with_encoder=False), n_lanes=lanes)
        rings["graph faster, %d lane(s)" % lanes] = FrameGraphRing(
            lambda: FrameGraph(net, faster, cal, "front", with_encoder=False), n_lanes=lanes)

    # ---- outputs first: the captured lossless frames (and the eager device loop) equal the eager engine bit for bit
    want = []
    for i in range(4):
        sdf, X, Y, Z, N = eager_frame(i)
        want.append((sdf.clone(), X, Y, Z, N, list(lossless.last_stats)))
    for i in range(4):
        got = eager_async_frame(i)
        for a, g in zip(want[i][:5], got):
            assert torch.equal(a, g), "eager device loop differs from the host-driven loop (frame %d)" % i
    for lanes in (1, 2):
        ring = rings["graph lossless, %d lane(s)" % lanes]
        for i, out in enumerate(ring.run(feats[i % 4] for i in range(4))):
            for a, g in zip(want[i][:5], out):
                assert torch.equal(a, g), "captured lossless frame differs from the eager engine (frame %d)" % i
            lane = ring.lanes[i % lanes]
            assert lane.last_stats == want[i][5]
            if lanes == 1:
                print("frame %d: %d points evaluated %s, conflict-loop passes per level %s"
                      % (i, sum(lane.last_stats), lane.last_stats, lane.last_conflict_loops))
    faster(im_feat_list=[[feats[0]]], calib_tensor=cal)
    print("faster frame 0: %d points evaluated %s" % (sum(faster.last_stats), faster.last_stats))
    print("outputs checked: the captured and eager-device-loop lossless frames equal the eager engine bit for bit")

    # ---- timing: warm-up, then alternating windows of at least args.window seconds
    def eager_variant(fn):
        def run(n):
            for i in range(n):
                fn(i)
        return run

    def ring_variant(ring):
        def run(n):
            for _ in ring.run(feats[i % 4] for i in range(n)):
                pass
        return run

    variants = {"eager lossless": eager_variant(eager_frame),
                "eager lossless, device loop": eager_variant(eager_async_frame)}
    for name, ring in rings.items():
        variants[name] = ring_variant(ring)
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
        print("%-32s %8.1f - %8.1f frames/s  (%6.3f - %6.3f ms/frame)" % (name, min(r), max(r), 1e3 / max(r), 1e3 / min(r)))
    for ring in rings.values():
        ring.close()
    torch.cuda.synchronize()
    lib.mp_octree_destroy(h)


if __name__ == "__main__":
    main()
