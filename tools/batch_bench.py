"""Batched query() and query_gradient() vs Python loops of single-image calls, on one GPU.

For the geometry head (256-channel maps) and the colour head (512-channel maps), B in {1, 2, 4, 8} images of 128 x 128 features
and N points per image in {5 000, 89 039 (the node count of one frame of the occupancy engine at its default levels),
1 000 000}: one `query()` over [B,C,H,W] / [B,3,N] / [B,4,4] (a single launch, mp_query_points_batch) against B calls of
`query()` with one image each.  Both variants upload their maps and rebuild the per-frame texel products (G0) on every call,
as a new frame would.  Times are CUDA-event medians after warm-up; every line reports the largest difference between the
batched and the looped outputs (the script stops above 1e-4).  The first line names the device and its power limit, read
in the same run.

--grad: the same comparison for `query_gradient()` (value and d points) in each precision of --precisions, for B in
{2, 4, 8} and N in {5 000, 100 000} by default: one batched call (mp_query_points_grad_batch: the calibs stay on the device)
against B single calls, each of which reads its camera back to the host; the loop is timed once as it is and once with
each call of the loop inside a `frame_scope()` (the batched call too), which is what an engine call does.  Both variants
again upload their maps and rebuild G0 on every call.

    python tools/batch_bench.py [--mode auto|tc|fp32] [--reps 5] [--warmup 2]
    python tools/batch_bench.py --grad [--precisions fp32,tc] [--batches 2,4,8] [--points 5000,100000]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

from oracle import spec  # noqa: E402
from helpers import build_net  # noqa: E402


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2], ts[0], ts[-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="auto", choices=["auto", "tc", "fp32"])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batches", default=None, help="default 1,2,4,8 (--grad: 2,4,8)")
    ap.add_argument("--points", default=None, help="default 5000,89039,1000000 (--grad: 5000,100000)")
    ap.add_argument("--grad", action="store_true", help="time query_gradient() instead of query()")
    ap.add_argument("--precisions", default="fp32,tc", help="--grad: the precisions of query_gradient() to time")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    props = torch.cuda.get_device_properties(0)
    print(json.dumps({"device": props.name, "sms": props.multi_processor_count, "power_limit_w": power_limit_w(),
                      "what": "query_gradient" if args.grad else "query", "mode": None if args.grad else args.mode,
                      "reps": args.reps, "warmup": args.warmup}), flush=True)
    Bs = [int(x) for x in (args.batches or ("2,4,8" if args.grad else "1,2,4,8")).split(",")]
    Ns = [int(x) for x in (args.points or ("5000,100000" if args.grad else "5000,89039,1000000")).split(",")]
    if args.grad:
        return grad_main(args, Bs, Ns)
    for head in ("G", "C"):
        chans = spec.G_CHANNELS if head == "G" else spec.C_CHANNELS
        Ws, bs = spec.make_weights(chans, 3 if head == "G" else 5)
        net = build_net(head, Ws, bs)
        net.precision = args.mode
        C = chans[0] - 1
        Bmax = max(Bs)
        feats = torch.cat([spec.make_feat(C, 128, 128, 40 + b, 0.5) for b in range(Bmax)], 0).cuda()
        cals = torch.cat([spec.scene_calib(20 + 10 * b, 33 - 15 * b) for b in range(Bmax)], 0).cuda()
        for N in Ns:
            pts_all = (torch.rand(Bmax, 3, N, generator=torch.Generator().manual_seed(N)) * 2.2 - 1.1).cuda()
            for B in Bs:
                f, p, c = feats[:B].contiguous(), pts_all[:B].contiguous(), cals[:B].contiguous()
                singles = [(f[b:b + 1], p[b:b + 1], c[b:b + 1]) for b in range(B)]
                res = {}

                def batched():
                    res["batched"] = net.query([[f]], p, calibs=c)[0]

                def looped():
                    res["looped"] = [net.query([[fb]], pb, calibs=cb)[0] for fb, pb, cb in singles]

                tb = timed(batched, args.reps, args.warmup)
                tl = timed(looped, args.reps, args.warmup)
                diff = (res["batched"] - torch.cat(res["looped"], 0)).abs().max().item()
                print(json.dumps({"head": head, "B": B, "N": N, "batched_ms": round(tb[0], 4), "looped_ms": round(tl[0], 4),
                                  "batched_ms_min_max": [round(tb[1], 4), round(tb[2], 4)],
                                  "looped_ms_min_max": [round(tl[1], 4), round(tl[2], 4)],
                                  "speedup": round(tl[0] / tb[0], 3),
                                  "batched_mpts_s": round(B * N / tb[0] / 1e3, 2), "equal": diff == 0.0,
                                  "max_abs_diff": diff}), flush=True)
                if diff > 1e-4:
                    raise SystemExit("batched output differs from the looped one (head %s B=%d N=%d)" % (head, B, N))


def grad_main(args, Bs, Ns):
    from monoport_b200 import _lib
    for head in ("G", "C"):
        chans = spec.G_CHANNELS if head == "G" else spec.C_CHANNELS
        Ws, bs = spec.make_weights(chans, 3 if head == "G" else 5)
        net = build_net(head, Ws, bs)
        C, R = chans[0] - 1, chans[-1]
        Bmax = max(Bs)
        feats = torch.cat([spec.make_feat(C, 128, 128, 40 + b, 0.5) for b in range(Bmax)], 0).cuda()
        cals = torch.cat([spec.scene_calib(20 + 10 * b, 33 - 15 * b) for b in range(Bmax)], 0).cuda()
        for precision in args.precisions.split(","):
            for N in Ns:
                pts_all = (torch.rand(Bmax, 3, N, generator=torch.Generator().manual_seed(N)) * 2.2 - 1.1).cuda()
                gout_all = torch.randn(Bmax, R, N, generator=torch.Generator().manual_seed(N + 1)).cuda()
                for B in Bs:
                    f, p, c, g = feats[:B].contiguous(), pts_all[:B].contiguous(), cals[:B].contiguous(), gout_all[:B].contiguous()
                    singles = [(f[b:b + 1], p[b:b + 1], c[b:b + 1], g[b:b + 1]) for b in range(B)]
                    res = {}

                    def batched():
                        res["batched"] = net.query_gradient([[f]], p, calibs=c, grad_output=g, precision=precision)

                    def looped():
                        res["looped"] = [net.query_gradient([[fb]], pb, calibs=cb, grad_output=gb, precision=precision)
                                         for fb, pb, cb, gb in singles]

                    def scoped(fn):
                        def run():
                            with _lib.frame_scope():
                                fn()
                        return run

                    tb = timed(batched, args.reps, args.warmup)
                    tl = timed(looped, args.reps, args.warmup)
                    diff = max((res["batched"][k] - torch.cat([r[k] for r in res["looped"]], 0)).abs().max().item()
                               for k in (0, 1))
                    tbs = timed(scoped(batched), args.reps, args.warmup)
                    tls = timed(scoped(looped), args.reps, args.warmup)
                    print(json.dumps({"head": head, "precision": precision, "B": B, "N": N,
                                      "batched_ms": round(tb[0], 4), "looped_ms": round(tl[0], 4),
                                      "batched_ms_min_max": [round(tb[1], 4), round(tb[2], 4)],
                                      "looped_ms_min_max": [round(tl[1], 4), round(tl[2], 4)],
                                      "speedup": round(tl[0] / tb[0], 3),
                                      "scoped_batched_ms": round(tbs[0], 4), "scoped_looped_ms": round(tls[0], 4),
                                      "scoped_speedup": round(tls[0] / tbs[0], 3),
                                      "batched_mpts_s": round(B * N / tb[0] / 1e3, 2), "equal": diff == 0.0,
                                      "max_abs_diff": diff}), flush=True)
                    if diff != 0.0:
                        raise SystemExit("batched gradient differs from the looped one (head %s %s B=%d N=%d)"
                                         % (head, precision, B, N))


if __name__ == "__main__":
    main()
