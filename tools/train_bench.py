"""Cost of the differentiable query for training (MonoPortNet.query_stages), on one GPU.

At PIFu training sizes -- B = 4 images of N = 5000 points, 128 x 128 feature maps -- forward plus backward (d features,
d points, d weights and d biases) of:
  vjp       MonoPortNet.query_stages: the exact fp32 query, then the fused sm_90a VJP kernel and the weight-gradient
            contraction (mp_query_points_vjp)
  autograd  the PyTorch restatement: index() (grid_sample) + the head's Conv1d forward, differentiated by autograd, TF32 off
for the geometry head over S = 4 hourglass stages (256-channel maps) and the colour head over one stage (512-channel maps).
Then one full training step of netG (PIFuHGFilters encoder on 4 x 3 x 512 x 512 images, 4 stages, MSE loss, SGD) with
query_stages, with the query's forward and backward timed alone on the same inputs, so its share of a step is visible.
Times are CUDA-event medians after warm-up.  The first line names the device, its power limit and its SM clock, read in
the same run.

--deterministic adds the ordered feature gradient (torch.use_deterministic_algorithms(True), MP_VJP_DETERMINISTIC): every
query_stages timing is then repeated `--rounds` times for each path, alternating the default (atomic) path and the ordered
one, and both are printed with the ordered path's cost relative to the default.  The full training step is timed with
the default path only (torch refuses the encoder's backward in deterministic mode).

    python tools/train_bench.py [--reps 10] [--warmup 3] [--deterministic [--rounds 3]]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from monoport_b200.modeling import PIFuNetC, PIFuNetG  # noqa: E402
from tools.batch_bench import power_limit_w, timed  # noqa: E402


def sm_clock_mhz():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def restated_query(net, feat, points, calibs):
    """index() + the head's forward, like the reference's train-mode query() for one stage"""
    xyz = net.projection(points, calibs)
    xy, z = xyz[:, :2, :], xyz[:, 2:3, :]
    in_img = (xy[:, 0] >= -1.0) & (xy[:, 0] <= 1.0) & (xy[:, 1] >= -1.0) & (xy[:, 1] <= 1.0)
    samples = F.grid_sample(feat, xy.transpose(1, 2).unsqueeze(2), align_corners=True)[:, :, :, 0]
    x = torch.cat([samples, z * net.normalizer.scale], 1)
    return in_img[:, None].float() * net.surface_classifier(x)


def query_inputs(net, C, S, B, N):
    g = torch.Generator(device="cuda").manual_seed(0)
    feats = [torch.randn(B, C, 128, 128, device="cuda", generator=g).requires_grad_() for _ in range(S)]
    points = (torch.rand(B, 3, N, device="cuda", generator=g) * 2 - 1).requires_grad_()
    calibs = torch.eye(4, device="cuda")[None].repeat(B, 1, 1)
    labels = torch.rand(B, net.surface_classifier.filter_channels[-1], N, device="cuda", generator=g)
    return feats, points, calibs, labels


def query_vjp_fn(net, C, S, B, N):
    """query_stages forward and backward of an MSE loss on query_case's inputs"""
    feats, points, calibs, labels = query_inputs(net, C, S, B, N)

    def vjp():
        preds = net.query_stages([[f] for f in feats], points, calibs)
        sum(F.mse_loss(p, labels) for p in preds).backward()
    return vjp


def query_case(net, C, S, B, N, reps, warmup):
    feats, points, calibs, labels = query_inputs(net, C, S, B, N)
    vjp = query_vjp_fn(net, C, S, B, N)

    def autograd():
        preds = [restated_query(net, f, points, calibs) for f in feats]
        sum(F.mse_loss(p, labels) for p in preds).backward()
    res = {}
    for name, fn in (("vjp", vjp), ("autograd", autograd)):
        res[name + "_ms"] = timed(fn, reps, warmup)[0]
    return res


def alternate(fn, reps, warmup, rounds):
    """medians of fn with torch's deterministic mode off and on, alternated `rounds` times -> dict(default_ms, ordered_ms
    (the median of the rounds' medians), their per-round lists and ordered / default)"""
    runs = {False: [], True: []}
    try:
        for _ in range(rounds):
            for det in (False, True):
                torch.use_deterministic_algorithms(det)
                runs[det].append(timed(fn, reps, warmup)[0])
    finally:
        torch.use_deterministic_algorithms(False)
    med = {k: sorted(v)[len(v) // 2] for k, v in runs.items()}
    return {"default_ms": round(med[False], 3), "ordered_ms": round(med[True], 3),
            "default_rounds_ms": [round(t, 3) for t in runs[False]], "ordered_rounds_ms": [round(t, 3) for t in runs[True]],
            "ordered_over_default": round(med[True] / med[False], 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--deterministic", action="store_true",
                    help="also time query_stages with the ordered feature gradient, alternating with the default path")
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    props = torch.cuda.get_device_properties(0)
    print(json.dumps({"device": props.name, "sms": props.multi_processor_count, "power_limit_w": power_limit_w(),
                      "sm_clock_mhz": sm_clock_mhz()}))
    B, N = 4, 5000
    netG = PIFuNetG().cuda().train()
    netC = PIFuNetC().cuda().train()
    for name, net, C, S in (("netG", netG, 256, 4), ("netC", netC, 512, 1)):
        r = query_case(net, C, S, B, N, a.reps, a.warmup)
        print(json.dumps({"case": "query fwd+bwd", "head": name, "B": B, "S": S, "N": N, **{k: round(v, 3) for k, v in r.items()},
                          "speedup": round(r["autograd_ms"] / r["vjp_ms"], 2)}))
        if a.deterministic:
            print(json.dumps({"case": "query fwd+bwd, ordered feature gradient", "head": name, "B": B, "S": S, "N": N,
                              **alternate(query_vjp_fn(net, C, S, B, N), a.reps, a.warmup, a.rounds)}))
    # one training step of netG: encoder, query_stages, loss, backward, SGD step
    g = torch.Generator(device="cuda").manual_seed(1)
    images = torch.randn(B, 3, 512, 512, device="cuda", generator=g)
    points = torch.rand(B, 3, N, device="cuda", generator=g) * 2 - 1
    calibs = torch.eye(4, device="cuda")[None].repeat(B, 1, 1)
    labels = torch.rand(B, 1, N, device="cuda", generator=g)
    opt = torch.optim.SGD(netG.parameters(), lr=1e-3)

    def step():
        opt.zero_grad()
        preds = netG.query_stages(netG.filter(images), points, calibs)
        netG.get_loss(preds, labels).backward()
        opt.step()
    t_step = timed(step, a.reps, a.warmup)[0]
    with torch.no_grad():
        stages = [[f.detach().clone().requires_grad_() for f in s] for s in netG.filter(images)]

    def query_only():
        preds = netG.query_stages(stages, points, calibs)
        netG.get_loss(preds, labels).backward()
    t_query = timed(query_only, a.reps, a.warmup)[0]
    print(json.dumps({"case": "netG training step", "B": B, "S": len(stages), "N": N, "step_ms": round(t_step, 3),
                      "query_fwd_bwd_ms": round(t_query, 3), "query_share": round(t_query / t_step, 3)}))
    if a.deterministic:
        print(json.dumps({"case": "netG training step's query fwd+bwd, ordered feature gradient", "B": B, "S": len(stages),
                          "N": N, **alternate(query_only, a.reps, a.warmup, a.rounds)}))


if __name__ == "__main__":
    main()
