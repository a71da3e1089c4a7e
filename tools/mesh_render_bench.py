"""What drawing the frame's mesh from viewer cameras costs (DESIGN.md §F3.2): bench.py's synthetic person at 257^3
(Seg3dLossless faster=True, features given, a seeded netC head on a 512-channel map), V in {1, 2, 4} views of the demo's
orthographic camera turned about the vertical axis, images of 256^2, 512^2 and 1024^2.

    python tools/mesh_render_bench.py [--rounds 3] [--window 1.0]

For every (V, size): eager recon.render_mesh of the frame's mesh with normals and colours, and the captured frame step
FrameGraph(mesh=True, mesh_normals=True, mesh_colours=True) with views= against the same graph without them; the render's
share of the frame is (with - without) / with.  Each variant is warmed up, then timed in synchronised windows of at least
`--window` seconds, the variants alternating round after round (median and range over the rounds).  Before anything is
timed, the captured images are checked against the eager render bit for bit.  The faces of the frame and the fragments of
view 0 (tests/raster_ref.py's count: covered pixel centres inside the depth range, before the depth test) are printed per
size.  The card's name and power limit are printed from the same run."""
import argparse
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))

VIEWS = (1, 2, 4)
SIZES = (256, 512, 1024)


def _views(V):
    import numpy as np
    from render_cases import demo_ortho, model
    return np.stack([model(0, 360.0 * k / V) for k in range(V)]), np.stack([demo_ortho()] * V)


def _timed(fn, window):
    import torch
    torch.cuda.synchronize()
    n, t0 = 0, time.perf_counter()
    while True:
        fn(n)
        n += 1
        torch.cuda.synchronize()
        if time.perf_counter() - t0 >= window:
            return (time.perf_counter() - t0) / n * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--window", type=float, default=1.0)
    args = ap.parse_args()
    import numpy as np
    import torch
    import bench
    import raster_ref
    from monoport_b200.engine import Seg3dLossless, make_query_func
    from monoport_b200.modeling import PIFuNetC, PIFuNetG
    from monoport_b200.pipeline import FrameGraph
    from monoport_b200.recon import mesh_colours, mesh_normals, reconstruction, render_mesh

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

    verts, faces, _, _ = reconstruction(net, dev, calg, R, b_min, b_max, use_octree=True, feats=[[feats[0]]], engine=eng)
    nrm = mesh_normals(net, [[feats[0]]], verts, calg, precision="auto")
    col = mesh_colours(netC, [[featsC[0]]], verts, calg)
    print("frame 0: %d vertices, %d faces per view" % (verts.shape[0], faces.shape[0]))
    vn, fn_, mats0 = verts.cpu().numpy(), faces.cpu().numpy(), raster_ref.view_mats(*_views(1))
    for S in SIZES:
        _, frags, listed = raster_ref.raster(vn, fn_, (len(vn), len(fn_)), mats0, S, S)
        print("%4d^2, view 0: %d fragments, %d covered pixels, %d faces on the large-face path"
              % (S, int(frags.sum()), int((frags > 0).sum()), listed))

    def graph(views=None, size=None):
        return FrameGraph(net, eng, cal, "front", with_encoder=False, netC=netC, mesh=True, mesh_normals=True,
                          mesh_colours=True, views=views, view_size=size)

    base = graph()
    for V in VIEWS:
        M, P = _views(V)
        for S in SIZES:
            g = graph((M, P), (S, S))
            g.launch(feats[0], featsC[0]).result()
            got = g.mesh_rendered()
            want = render_mesh(verts, faces, M, P, (S, S), normals=nrm, colours=col)
            assert all(torch.equal(torch.nan_to_num(a), torch.nan_to_num(w)) for a, w in zip(got, want)), (V, S)

            def eager(i):
                render_mesh(verts, faces, M, P, (S, S), normals=nrm, colours=col)

            def with_views(i):
                g.launch(feats[i % 4], featsC[i % 4]).result()

            def without(i):
                base.launch(feats[i % 4], featsC[i % 4]).result()
            fns = {"eager render_mesh": eager, "frame with views": with_views, "frame without views": without}
            times = {k: [] for k in fns}
            for f in fns.values():
                f(0)
                f(1)
            for _ in range(args.rounds):
                for k, f in fns.items():
                    times[k].append(_timed(f, args.window))
            med = {k: statistics.median(t) for k, t in times.items()}
            print("V=%d %4d^2: " % (V, S) + "; ".join("%s %.3f ms (%.3f-%.3f)" % (k, med[k], min(t), max(t))
                                                      for k, t in times.items())
                  + "; render share of the frame %.1f %%" % (100 * (med["frame with views"] - med["frame without views"])
                                                              / med["frame with views"]))
            g.close()
    base.close()


if __name__ == "__main__":
    main()
