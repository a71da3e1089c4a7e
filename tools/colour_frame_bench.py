"""What the demo's whole frame costs -- geometry, the normal image and the netC colour image (RTL/main.py:417-441) --
eager against the captured frame step (pipeline.FrameGraph with netC and render_normals, FrameGraphRing at 1, 2 and 4
lanes), with the features given and with both encoders (HG for netG, ResBlk for netC with netG's map as its prior).
The geometry-only captured graph is timed beside them, and so is the captured frame whose normal image comes from the
geometry net's analytic normals (render_normals="gradient": the tensor-core gradient, mp_surface_normals_async) instead
of forward_vertices' finite differences.  Workload: bench.py's synthetic person, 257^3 Seg3dLossless
(faster=True), a seeded netC head on a 512-channel map.

    python tools/colour_frame_bench.py [--rounds 3] [--window 1.0]

Outputs are compared before anything is timed.  Every variant is warmed up, then timed in synchronised windows of at least
`--window` seconds, the variants alternating round after round; the line of a variant gives the range over the rounds.
The card's name and power limit are printed from the same run."""
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
    net.image_filter.to(dev)
    net.eval()
    netC = PIFuNetC()
    netC.to(dev)
    netC.eval()
    feats = [f.to(dev) for f in feats_cpu]
    gC = torch.Generator().manual_seed(11)
    featsC = [(torch.randn(1, 512, 128, 128, generator=gC) * 0.5).to(dev) for _ in range(4)]
    gI = torch.Generator().manual_seed(5)
    imgs = [(torch.rand(1, 3, 512, 512, generator=gI) * 2 - 1).to(dev) for _ in range(4)]
    imgsC = [(torch.rand(1, 3, 512, 512, generator=gI) * 2 - 1).to(dev) for _ in range(4)]
    hook = bench._person_hook(feats[0][:, 0].clone())
    cal = bench.scene_calib()
    b = np.array([bench.B_MIN], dtype=np.float32)
    eng = Seg3dLossless(make_query_func(net), b, -b, [17, 33, 65, 129, 257], balance_value=0.5, faster=True).to(dev)
    R = 257
    calg = cal.to(dev)

    @torch.no_grad()
    def eager_frame(i, encoders):
        if encoders:
            fe = hook(net.filter(imgs[i % 4])[-1][0])
            fc = netC.filter(imgsC[i % 4], feat_prior=fe)[-1][0]
        else:
            fe, fc = feats[i % 4], featsC[i % 4]
        sdf = eng(im_feat_list=[[fe]], calib_tensor=cal)
        X, Y, Z, N = forward_vertices(sdf, "front")
        rn = colorization(netC, None, X, Y, Z, calg, norm=N, resolution=R)
        rt = colorization(netC, [[fc]], X, Y, Z, calg, resolution=R)
        return sdf, X, rn, rt

    def items(encoders, n):
        if encoders:
            return ((imgs[i % 4], imgsC[i % 4]) for i in range(n))
        return ((feats[i % 4], featsC[i % 4]) for i in range(n))

    rings = {}
    for lanes in (1, 2, 4):
        rings["graph geometry only, %d lane(s)" % lanes] = (FrameGraphRing(
            lambda: FrameGraph(net, eng, cal, "front", with_encoder=False), n_lanes=lanes), lambda n: (feats[i % 4] for i in range(n)))
        for enc in (False, True):
            rings["graph + normals + colour, %s, %d lane(s)" % ("encoders" if enc else "features given", lanes)] = (FrameGraphRing(
                lambda: FrameGraph(net, eng, cal, "front", with_encoder=enc, feature_hook=hook if enc else None, netC=netC,
                                   render_normals=True), n_lanes=lanes), (lambda e: lambda n: items(e, n))(enc))
        rings["graph + analytic normals + colour, features given, %d lane(s)" % lanes] = (FrameGraphRing(
            lambda: FrameGraph(net, eng, cal, "front", with_encoder=False, netC=netC, render_normals="gradient"),
            n_lanes=lanes), lambda n: items(False, n))

    # ---- the outputs first: the captured frames equal the eager chain (features given: bit for bit; encoders: the set
    # pixels, and the values to the encoders' float noise under capture)
    for enc in (False, True):
        want = [eager_frame(i, enc) for i in range(4)]
        for lanes in (1, 2, 4):
            ring, _ = rings["graph + normals + colour, %s, %d lane(s)" % ("encoders" if enc else "features given", lanes)]
            for i, out in enumerate(ring.run(items(enc, 4))):
                sdf, X, rn, rt = want[i]
                if not enc:
                    assert torch.equal(out[0], sdf) and torch.equal(out[1], X), "geometry differs"
                    assert torch.equal(out[5], rn) and torch.equal(out[6], rt), "images differ"
                else:
                    set_g, set_e = (out[6] != 1.0).any(-1), (rt != 1.0).any(-1)
                    print("encoders, %d lane(s), frame %d: %d / %d colour pixels set in both, max|graph - eager| %.2e"
                          % (lanes, i, int((set_g & set_e).sum()), int(set_e.sum()), (out[6] - rt)[set_g & set_e].abs().max().item()))
    for lanes in (1, 2, 4):
        ring, _ = rings["graph + analytic normals + colour, features given, %d lane(s)" % lanes]
        for i, out in enumerate(ring.run(items(False, 4))):
            sdf = eng(im_feat_list=[[feats[i % 4]]], calib_tensor=cal)
            X, Y, Z, _ = forward_vertices(sdf, "front")
            nrm = surface_normals(net, [[feats[i % 4]]], X, Y, Z, calg, resolution=R, precision="auto")
            assert torch.equal(out[5], colorization(None, None, X, Y, Z, calg, norm=nrm, resolution=R)), "analytic normal image differs"
    print("outputs checked: the captured frames equal the eager chain")

    # ---- timing: warm-up, then alternating windows of at least args.window seconds
    def eager_variant(enc):
        def run(n):
            for i in range(n):
                eager_frame(i, enc)
        return run

    def ring_variant(ring, gen):
        def run(n):
            for _ in ring.run(gen(n)):
                pass
        return run

    variants = {"eager chain, features given": eager_variant(False), "eager chain, encoders": eager_variant(True)}
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
