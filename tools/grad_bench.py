"""Cost of the point gradient of query(), on one GPU.

For the geometry head (256-channel maps) and the colour head (512-channel maps) on 128 x 128 features, N in {10^4, 10^5,
10^6} random points seen by the demo camera, in one call:
  grad      MonoPortNet.query_gradient (value + gradient, one launch of the fp32 gradient kernel)
  grad-tc   MonoPortNet.query_gradient with precision "tc" (the tensor-core program's forward-mode derivative; its
            per-frame texel products are rebuilt every call).  grad and grad-tc are timed twice, alternated, and the
            faster round of each is reported
  fp32      query() with precision "fp32" (the forward half alone, the same CUDA-core arithmetic)
  tc        query() with precision "tc" (the tensor-core program; its per-frame texel products are rebuilt every call)
  autograd  a PyTorch restatement in this file: grid_sample + matmuls + autograd on the GPU, fp32
Times are CUDA-event medians after warm-up.  The useful FLOPs are computed from the head's shapes: 2 * sum(cin * cout) per
point for the forward MLP and as much again for the reverse pass (the transposed products); sampling is not counted.
Every line also reports the largest difference of the gradient against the autograd restatement, relative to its largest
entry, and the fraction of components within 2e-5 of that entry (single outliers come from leaky-ReLU and texel kinks, where
fp32 rounding decides the side).  Last, reconstruction() of the synthetic person at 257^3 (dense grid query, marching cubes) with normals=False and
normals=True (the grid query in the default "auto" precision).  The first line names the device and its power limit, read in the same run.

    python tools/grad_bench.py [--reps 5] [--warmup 2] [--points 10000,100000,1000000]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from oracle import spec  # noqa: E402
from helpers import build_net  # noqa: E402
from tools.batch_bench import power_limit_w, timed  # noqa: E402


def autograd_query(feat, points, calib, Ws, bs, last_op, z_scale=spec.Z_SCALE):
    """query() for B = 1 as PyTorch ops (orthogonal projection, grid_sample, 1x1 convolutions as matmuls) and its gradient
    with respect to the points by autograd: -> (value [Res,N], dpoints [3,N])"""
    p = points.detach().requires_grad_(True)
    xyz = calib[:3, :3] @ p + calib[:3, 3:4]
    u, v, z = xyz[0], xyz[1], xyz[2]
    in_img = ((u >= -1) & (u <= 1) & (v >= -1) & (v <= 1)).float()
    grid = torch.stack([u, v], 1)[None, :, None, :]                               # [1,N,1,2]
    x = F.grid_sample(feat, grid, align_corners=True)[0, :, :, 0]                 # [C,N]
    x = torch.cat([x, (z * z_scale)[None]], 0)
    y = x
    for l, (W, b) in enumerate(zip(Ws, bs)):
        y = torch.addmm(b[:, None], W, y if l == 0 else torch.cat([y, x], 0))
        if l != len(Ws) - 1:
            y = F.leaky_relu(y, spec.LEAKY_SLOPE)
    y = torch.sigmoid(y) if last_op == spec.LAST_SIGMOID else torch.tanh(y)
    out = in_img[None] * y
    (dp,) = torch.autograd.grad(out, p, grad_outputs=torch.ones_like(out))
    return out.detach(), dp


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--points", default="10000,100000,1000000")
    ap.add_argument("--recon-res", type=int, default=257)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("grad_bench needs a CUDA device")
    torch.cuda.set_device(0)
    props = torch.cuda.get_device_properties(0)
    print(json.dumps({"device": props.name, "sms": props.multi_processor_count, "power_limit_w": power_limit_w(),
                      "reps": args.reps, "warmup": args.warmup}), flush=True)
    cal = spec.scene_calib(20, 33).cuda()
    for head in ("G", "C"):
        chans = spec.G_CHANNELS if head == "G" else spec.C_CHANNELS
        last_op = spec.LAST_SIGMOID if head == "G" else spec.LAST_TANH
        Ws, bs = spec.make_weights(chans, 3 if head == "G" else 5)
        net = build_net(head, Ws, bs)
        Wd, bd = [w.cuda() for w in Ws], [b.cuda() for b in bs]
        feat = spec.make_feat(chans[0] - 1, 128, 128, 4, 0.5).cuda()
        feats = [[feat]]
        mlp_flop = 2 * sum(w.shape[0] * w.shape[1] for w in Ws)                 # per point, one direction
        tc_ok = net.surface_classifier.tc_supported()
        for N in (int(x) for x in args.points.split(",")):
            pts = (torch.rand(1, 3, N, generator=torch.Generator().manual_seed(N)) * 2.2 - 1.1).cuda()
            res = {}

            def grad():
                res["grad"] = net.query_gradient(feats, pts, calibs=cal)

            def grad_tc():
                res["grad_tc"] = net.query_gradient(feats, pts, calibs=cal, precision="tc")

            def fp32():
                net.precision = "fp32"
                net.query(feats, pts, calibs=cal)

            def tc():
                net.precision = "tc"
                net.query(feats, pts, calibs=cal)

            def autograd():
                res["autograd"] = autograd_query(feat, pts[0], cal[0], Wd, bd, last_op)

            t = {"grad": timed(grad, args.reps, args.warmup), "fp32": timed(fp32, args.reps, args.warmup),
                 "autograd": timed(autograd, args.reps, args.warmup)}
            if tc_ok:
                t["tc"] = timed(tc, args.reps, args.warmup)
                t["grad_tc"] = timed(grad_tc, args.reps, args.warmup)
                g2 = timed(grad, args.reps, args.warmup)
                t["grad"] = min(t["grad"], g2)
                t["grad_tc"] = min(t["grad_tc"], timed(grad_tc, args.reps, args.warmup))
            ref = res["autograd"][1]
            err = (res["grad"][1][0] - ref).abs() / ref.abs().max()
            rel = err.max().item()
            frac = (err <= 2e-5).double().mean().item()
            line = {"head": head, "N": N, "mlp_mflop_per_point_fwd": round(mlp_flop / 1e6, 4)}
            for k, (med, lo, hi) in t.items():
                line[k + "_ms"] = round(med, 4)
                line[k + "_ms_min_max"] = [round(lo, 4), round(hi, 4)]
            line["grad_mpts_s"] = round(N / t["grad"][0] / 1e3, 2)
            line["grad_tflop_s"] = round(2 * mlp_flop * N / t["grad"][0] / 1e9, 2)
            line["fp32_tflop_s"] = round(mlp_flop * N / t["fp32"][0] / 1e9, 2)
            line["grad_over_fp32"] = round(t["grad"][0] / t["fp32"][0], 3)
            line["autograd_over_grad"] = round(t["autograd"][0] / t["grad"][0], 3)
            line["max_rel_diff_vs_autograd"] = rel
            line["frac_within_2e-5_of_max_vs_autograd"] = round(frac, 6)
            if tc_ok:
                line["grad_tc_mpts_s"] = round(N / t["grad_tc"][0] / 1e3, 2)
                line["grad_tc_speedup_over_grad"] = round(t["grad"][0] / t["grad_tc"][0], 2)
                etc = (res["grad_tc"][1][0] - ref).abs() / ref.abs().max()
                line["grad_tc_rel_diff_vs_autograd_median_p99_max"] = [etc.median().item(), etc.quantile(0.99).item()
                                                                       if etc.numel() <= 1 << 24 else None, etc.max().item()]
            print(json.dumps(line), flush=True)
            del res
            torch.cuda.empty_cache()
    # reconstruction of the synthetic person with and without normals
    from monoport_b200.recon import reconstruction
    Ws, bs = spec.make_weights(spec.G_CHANNELS, 3)
    feat = spec.make_feat(256, 128, 128, 4, 0.5)
    Ws, bs, feat, _ = spec.heightfield_person(Ws, bs, feat)
    net = build_net("G", Ws, bs)
    net.precision = "auto"
    feats = [[feat.cuda()]]
    R = args.recon_res
    cal = spec.scene_calib(20, 0).cuda()
    out = {}

    def recon(normals):
        def f():
            out[normals] = reconstruction(net, "cuda:0", cal, R, [-1, -1, -1], [1, 1, 1], feats=feats, normals=normals)
        return f

    t0 = timed(recon(False), args.reps, args.warmup)
    t1 = timed(recon(True), args.reps, args.warmup)
    print(json.dumps({"reconstruction_R": R, "query": net.precision, "vertices": int(out[True][0].shape[0]),
                      "normals_false_ms": round(t0[0], 3), "normals_true_ms": round(t1[0], 3),
                      "normals_false_ms_min_max": [round(t0[1], 3), round(t0[2], 3)],
                      "normals_true_ms_min_max": [round(t1[1], 3), round(t1[2], 3)],
                      "normals_extra_ms": round(t1[0] - t0[0], 3)}), flush=True)


if __name__ == "__main__":
    main()
