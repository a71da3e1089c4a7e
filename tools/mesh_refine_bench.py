"""What the mesh refinement costs and buys (DESIGN.md §F3.1): a 257^3 frame of bench.py's synthetic person through
pipeline.FrameGraph(mesh=True, mesh_refine=K) and eager reconstruction(use_octree=True, engine=..., refine=K), K in {0, 2, 4}
(Seg3dLossless faster=True, features given, the net's default precision), and the accuracy of the vertices against a float64
evaluation of the head on dense R = 129 and R = 257 volumes.

    python tools/mesh_refine_bench.py [--rounds 3] [--window 1.0] [--accuracy-rounds 4]

Timing: every variant is warmed up, then timed in synchronised windows of at least `--window` seconds, the variants
alternating round after round; a line gives ms per frame (median and range over the rounds), ms per refinement round against
K = 0 of the same kind, and the frame's vertex count.  Before anything is timed, the captured mesh of every K is checked
against the eager one bit for bit.
Accuracy: over the vertices whose float64 end values bracket iso, p50 / p99 / max of |sigma64(v) - iso| and of the distance
along the edge (in voxels) to the float64 root of the head, for the marching-cubes and the refined vertices.
The card's name and power limit are printed from the same run."""
import argparse
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))

KS = (0, 2, 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--accuracy-rounds", type=int, default=4)
    args = ap.parse_args()
    import numpy as np
    import torch
    import bench
    from mesh_refine_ref import edge_parameter, edge_roots64, query64
    from monoport_b200.engine import Seg3dLossless, make_query_func
    from monoport_b200.modeling import PIFuNetG
    from monoport_b200.pipeline import FrameGraph
    from monoport_b200.recon import McubesWorkspace, marching_cubes_async, reconstruction, refine_mesh_async

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
    calg = bench.scene_calib().to(dev)
    b = np.array([bench.B_MIN], dtype=np.float32)
    eng = Seg3dLossless(make_query_func(net), b, -b, [17, 33, 65, 129, 257], balance_value=0.5, faster=True).to(dev)
    R = 257
    b_min, b_max = b[0], -b[0]

    graphs = {K: FrameGraph(net, eng, bench.scene_calib(), "front", with_encoder=False, mesh=True, mesh_refine=K) for K in KS}

    @torch.no_grad()
    def eager(i, K):
        r = reconstruction(net, dev, calg, R, b_min, b_max, use_octree=True, feats=[[feats[i % 4]]], engine=eng, refine=K)
        return None if isinstance(r, int) else r[:2]

    def captured(i, K):
        g = graphs[K]
        g.launch(feats[i % 4]).result()
        return g.mesh()

    n_verts = {}
    for K in KS:
        for i in range(4):
            w, got = eager(i, K), captured(i, K)
            assert torch.equal(w[0], got[0]) and torch.equal(w[1], got[1]), (K, i)
        n_verts[K] = int(w[0].shape[0])
    print("captured meshes equal the eager chain bit for bit for K in %s; frame 3 has %d vertices" % (KS, n_verts[0]))

    variants = [("graph", K) for K in KS] + [("eager", K) for K in KS]
    times = {v: [] for v in variants}
    for _ in range(2):
        for kind, K in variants:
            (captured if kind == "graph" else eager)(0, K)
    for _ in range(args.rounds):
        for kind, K in variants:
            fn = captured if kind == "graph" else eager
            torch.cuda.synchronize()
            n, t0 = 0, time.perf_counter()
            while True:
                fn(n, K)
                n += 1
                torch.cuda.synchronize()
                if time.perf_counter() - t0 >= args.window:
                    break
            times[(kind, K)].append((time.perf_counter() - t0) / n * 1e3)
    for kind, K in variants:
        med = statistics.median(times[(kind, K)])
        base = statistics.median(times[(kind, 0)])
        per_round = "" if K == 0 else ", %.3f ms per round" % ((med - base) / K)
        print("%-5s mesh_refine=%d: %.3f ms per frame (%.3f-%.3f)%s, %d vertices"
              % (kind, K, med, min(times[(kind, K)]), max(times[(kind, K)]), per_round, n_verts[K]))
    for g in graphs.values():
        g.close()

    # ---- accuracy on dense volumes
    K = args.accuracy_rounds
    Wd, bd = [w.to(dev) for w in Ws], [x.to(dev) for x in bs]
    feat = feats[0]

    def s64(p):
        return query64(feat, p.to(dev), calg, Wd, bd)[0]
    for Rv in (129, 257):
        vol = net.query_grid(feat, calg, Rv, torch.tensor(b_min), torch.tensor(b_max))
        ws = McubesWorkspace(vol.shape, dev)
        cap = 8 * Rv * Rv
        verts = torch.empty((cap, 3), device=dev)
        faces = torch.empty((2 * cap, 3), dtype=torch.int32, device=dev)
        counts = torch.zeros(2, dtype=torch.int64, device=dev)
        c32 = torch.zeros(1, dtype=torch.int32, device=dev)
        marching_cubes_async(vol, verts, faces, counts, c32, 0.5, b_min, b_max, workspace=ws)
        torch.cuda.synchronize()
        nv = int(counts[0])
        assert nv <= cap
        mc = verts[:nv].clone()
        refine_mesh_async(net, feat, vol, verts, c32, K, b_min, b_max, calg, workspace=ws)
        torch.cuda.synchronize()
        ws.close()
        ref = verts[:nv].clone()
        v = vol.cpu().numpy()
        mask, t_root = edge_roots64(s64, v, 0.5, b_min, b_max)
        rows = []
        for name, x in (("MC", mc), ("refined K=%d" % K, ref)):
            e = (s64(x.double().t()).cpu() - 0.5).abs()[mask]
            d = (edge_parameter(x, v, 0.5, b_min, b_max) - t_root).abs()[mask]
            q = torch.tensor([0.5, 0.99], dtype=torch.float64)
            rows.append("  %-13s |sigma64 - iso| p50 %.3e p99 %.3e max %.3e;  edge distance to the root (voxels) p50 %.3e "
                        "p99 %.3e max %.3e" % (name, *torch.quantile(e, q).tolist(), e.max().item(),
                                               *torch.quantile(d, q).tolist(), d.max().item()))
        print("R=%d (%s): %d vertices, %d bracketed in float64" % (Rv, net.precision, nv, int(mask.sum())))
        print("\n".join(rows))


if __name__ == "__main__":
    main()
