"""What a mesh per frame costs: the eager chain (reconstruction(use_octree=True, engine=...) = engine + marching cubes + world
mapping, then mesh_normals(precision="auto") and mesh_colours with netC) against the captured frame step
(pipeline.FrameGraph(mesh=True[, mesh_normals=True, mesh_colours=True]), FrameGraphRing at 1, 2 and 4 lanes).  The
geometry-only captured graph (no mesh) is timed beside them.  Workload: bench.py's synthetic person, 257^3 Seg3dLossless
(faster=True), features given, a seeded netC head on a 512-channel map.

    python tools/mesh_frame_bench.py [--rounds 3] [--window 1.0]

Outputs are compared before anything is timed: every lane count's captured mesh, normals and colours equal the eager
chain's bit for bit.  Every variant is warmed up, then timed in synchronised windows of at least `--window` seconds, the
variants alternating round after round; the line of a variant gives the range over the rounds.  The card's name and power
limit are printed from the same run."""
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
    from monoport_b200.engine import Seg3dLossless, make_query_func
    from monoport_b200.modeling import PIFuNetC, PIFuNetG
    from monoport_b200.pipeline import FrameGraph, FrameGraphRing
    from monoport_b200.recon import mesh_colours, mesh_normals, reconstruction

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
    cal = bench.scene_calib()
    calg = cal.to(dev)
    b = np.array([bench.B_MIN], dtype=np.float32)
    eng = Seg3dLossless(make_query_func(net), b, -b, [17, 33, 65, 129, 257], balance_value=0.5, faster=True).to(dev)
    R = 257
    b_min, b_max = b[0], -b[0]

    @torch.no_grad()
    def eager_frame(i, extras):
        r = reconstruction(net, dev, calg, R, b_min, b_max, use_octree=True, feats=[[feats[i % 4]]], engine=eng)
        if isinstance(r, int):
            return None
        verts, faces, _, _ = r
        if not extras:
            return verts, faces
        return (verts, faces, mesh_normals(net, [[feats[i % 4]]], verts, calg, precision="auto"),
                mesh_colours(netC, [[featsC[i % 4]]], verts, calg))

    def items(n):
        return ((feats[i % 4], featsC[i % 4]) for i in range(n))

    rings = {}
    for lanes in (1, 2, 4):
        rings["graph geometry only, %d lane(s)" % lanes] = (FrameGraphRing(
            lambda: FrameGraph(net, eng, cal, "front", with_encoder=False), n_lanes=lanes), lambda n: (feats[i % 4] for i in range(n)))
        rings["graph + mesh, %d lane(s)" % lanes] = (FrameGraphRing(
            lambda: FrameGraph(net, eng, cal, "front", with_encoder=False, mesh=True), n_lanes=lanes),
            lambda n: (feats[i % 4] for i in range(n)))
        rings["graph + mesh + normals + colours, %d lane(s)" % lanes] = (FrameGraphRing(
            lambda: FrameGraph(net, eng, cal, "front", with_encoder=False, netC=netC, mesh=True, mesh_normals=True,
                               mesh_colours=True), n_lanes=lanes), items)

    # ---- the outputs first: the captured meshes equal the eager chain bit for bit
    want = [eager_frame(i, True) for i in range(4)]
    for i, w in enumerate(want):
        print("frame %d: %d vertices, %d faces" % (i, w[0].shape[0], w[1].shape[0]))
    for lanes in (1, 2, 4):
        ring, gen = rings["graph + mesh + normals + colours, %d lane(s)" % lanes]
        for i, out in enumerate(ring.run(gen(4))):
            for a, g in zip(want[i], out[7:]):
                assert a.shape == g.shape and torch.equal(a, g), "captured mesh differs (frame %d, %d lanes)" % (i, lanes)
        ring, gen = rings["graph + mesh, %d lane(s)" % lanes]
        for i, out in enumerate(ring.run(gen(4))):
            assert torch.equal(out[5], want[i][0]) and torch.equal(out[6], want[i][1]) and out[7] is None and out[8] is None
    print("outputs checked: the captured meshes equal the eager chain")

    # ---- timing: warm-up, then alternating windows of at least args.window seconds
    def eager_variant(extras):
        def run(n):
            for i in range(n):
                eager_frame(i, extras)
        return run

    def ring_variant(ring, gen):
        def run(n):
            for _ in ring.run(gen(n)):
                pass
        return run

    variants = {"eager mesh chain, geometry only": eager_variant(False),
                "eager mesh chain + normals + colours": eager_variant(True)}
    for name, (ring, gen) in rings.items():
        variants[name] = ring_variant(ring, gen)
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
