"""The differentiable query for training (MonoPortNet.query_stages -> mp_query_points_vjp): a float64 / float32 restatement of
the reference's train-mode query() differentiated by autograd (`query_vjp_ref`), the error bar of its gradients, the
reference goldens (tests/golden/vjp_*.npz, tests/golden/make_vjp_golden.py), the regeneration of their seeded inputs, and
the backward of one stage on the CPU model (`run_vjp`)."""
import glob
import os

import numpy as np
import torch
import torch.nn as nn

from oracle import spec
from emu_harness import run
from helpers import GOLDEN

GRAD_NAMES = ("dfeat", "dpoints", "dW", "db")


def query_vjp_ref(feats, points, calib, Ws, bs, last_op, proj="orthogonal", grad_output=None, dtype=torch.float64,
                  z_scale=spec.Z_SCALE):
    """The reference's train-mode query() (MonoPortNet.py:63-91) restated from the oracle's pieces, differentiated by autograd
    in `dtype`.  feats: S maps [B,C,H,W] (one per stage); points [B,3,N]; calib [B,4,4]|[B,3,4]|None; grad_output: S
    tensors [B,Res,N] or None (ones).  -> dict(value [S][B,Res,N], dfeat [S][B,C,H,W], dpoints [B,3,N], dW [L], db [L]) of
    sum_s sum(grad_output_s * value_s)."""
    fs = [f.to(dtype).detach().clone().requires_grad_() for f in feats]
    p = points.to(dtype).detach().clone().requires_grad_()
    Wt = [w.to(dtype).detach().clone().requires_grad_() for w in Ws]
    bt = [b.to(dtype).detach().clone().requires_grad_() for b in bs]
    B = p.shape[0]
    with torch.enable_grad():
        values = []
        for f in fs:
            outs = []
            for b in range(B):
                xyz = spec.project_ref(p[b], None if calib is None else calib[b].to(dtype), proj)
                u, v, z = xyz[0], xyz[1], xyz[2]
                in_img = (u >= -1.0) & (u <= 1.0) & (v >= -1.0) & (v <= 1.0)
                x = torch.cat([spec.bilinear_ref(f[b], u, v), (z * z_scale)[None]], 0)
                outs.append(in_img.to(dtype)[None] * spec.mlp_ref(x, Wt, bt, last_op))
            values.append(torch.stack(outs))
        total = sum((v * (torch.ones_like(v) if grad_output is None else grad_output[s].to(dtype))).sum()
                    for s, v in enumerate(values))
        grads = torch.autograd.grad(total, fs + [p] + Wt + bt)
    S, L = len(fs), len(Ws)
    return dict(value=[v.detach() for v in values], dfeat=list(grads[:S]), dpoints=grads[S],
                dW=list(grads[S + 1:S + 1 + L]), db=list(grads[S + 1 + L:]))


def flat(ts):
    """one flat float64 vector of a tensor or a list of tensors"""
    if isinstance(ts, (list, tuple)):
        return torch.cat([t.detach().double().reshape(-1).cpu() for t in ts])
    return ts.detach().double().reshape(-1).cpu()


def vjp_bar(got, g64, ref32_dist=0.0):
    """The error bar of a gradient against the reference's fp64 one (F1'''s convention): every component within
    max(1e-3, 1.1 * ref32_dist) * max|g64| -- ref32_dist the reference fp32 gradient's own largest distance, relative -- and
    99 % of them within 2e-5 * max|g64|.  Tensors or lists of tensors.  -> (ok, message)"""
    got, g64 = flat(got), flat(g64)
    scale = g64.abs().max().item()
    if scale == 0.0:
        return bool((got == 0).all()), "reference gradient is zero, max|got| = %.2e" % got.abs().max().item()
    err = (got - g64).abs() / scale
    worst, frac = err.max().item(), (err <= 2e-5).double().mean().item()
    bar = max(1e-3, 1.1 * ref32_dist)
    return worst <= bar and frac >= 0.99, "max|err|/max|g| = %.2e (bar %.2e), fraction within 2e-5: %.4f" % (worst, bar, frac)


def rel_dist(a, b64):
    """max|a - b64| / max|b64| over tensors or lists of tensors"""
    a, b64 = flat(a), flat(b64)
    return ((a - b64).abs().max() / b64.abs().max().clamp_min(1e-300)).item()


# ---- the reference goldens -------------------------------------------------------------------------------------------------
def vjp_cases():
    return sorted(os.path.basename(p)[len("vjp_"):-4] for p in glob.glob(os.path.join(GOLDEN, "vjp_*.npz")))


def sample_index(numel, seed, k=4096):
    """the seeded components a golden stores of a gradient with `numel` components (all of them when there are at most k)"""
    if numel <= k:
        return torch.arange(numel)
    return torch.randperm(numel, generator=torch.Generator().manual_seed(seed))[:k].sort().values


def case_calib(kind, b):
    """the camera of image b of a golden: "rot" (orthographic, rotated), "persp" (perspective) or "none" -> [4,4] | None"""
    if kind == "none":
        return None
    c = spec.scene_calib(20.0 + 10.0 * b, 33.0 - 7.0 * b)[0].clone()
    if kind == "persp":
        c[2, 3] = 3.0          # z away from 0, so that x/z, y/z stay finite and mostly in the image
        c[:2, :] *= 2.5
    return c


def case_points(N, seed):
    """[3,N] seeded points, the first 8 on the image border / corners and far outside"""
    p = spec.make_points(N, seed)[0].clone()
    if N >= 16:
        p[:, :8] = torch.tensor([[1.0, -1.0, 1.0, 0.0, 5.0, 0.0, -1.0, 1.0000001],
                                 [0.3, -1.0, 1.0, 1.0, 0.0, 0.0, 0.999999, 0.0],
                                 [0.1, 0.0, -0.5, 0.9, 0.0, 0.0, 0.2, 0.2]])
    return p


def make_case_inputs(c):
    """the seeded inputs of a golden's parameters `c` (mapping: chans, wseed, fseed, pseed, gseed, B, S, N, H, W, calib,
    proj, last_op) -> dict(feats [S][B,C,H,W], points [B,3,N], calib [B,4,4]|None, Ws, bs, grad_output [S][B,Res,N]|None)"""
    chans = [int(x) for x in c["chans"]]
    Ws, bs = spec.make_weights(chans, int(c["wseed"]))
    B, S, N, H, W = (int(c[k]) for k in ("B", "S", "N", "H", "W"))
    feats = [torch.cat([spec.make_feat(chans[0] - 1, H, W, int(c["fseed"]) + 100 * s + b) for b in range(B)])
             for s in range(S)]
    points = torch.stack([case_points(N, int(c["pseed"]) + b) for b in range(B)])
    kind = str(c["calib"])
    cal = None if kind == "none" else torch.stack([case_calib(kind, b) for b in range(B)])
    gout = None
    if int(c["gseed"]) >= 0:
        g = torch.Generator().manual_seed(int(c["gseed"]))
        gout = [torch.randn(B, chans[-1], N, generator=g) for _ in range(S)]
    last_op = {"sigmoid": spec.LAST_SIGMOID, "tanh": spec.LAST_TANH, "none": spec.LAST_NONE}[str(c["last_op"])]
    return dict(feats=feats, points=points, calib=cal, Ws=Ws, bs=bs, grad_output=gout, last_op=last_op, chans=chans,
                proj="perspective" if kind == "persp" else "orthogonal")


def load_vjp_case(name):
    """-> the inputs (make_case_inputs) and, per gradient g in GRAD_NAMES: idx_g (the stored components of the flattened
    gradient -- dfeat: all stages, dW / db: all layers, concatenated), g64 / g32 (the reference's fp64 / fp32 values there),
    scale_g (max|g64| over every component) and dist_g (the reference fp32 gradient's largest distance from its fp64 one
    over every component, relative to scale_g)"""
    z = np.load(os.path.join(GOLDEN, "vjp_%s.npz" % name))
    c = make_case_inputs(z)
    c["name"] = name
    for g in GRAD_NAMES:
        c["idx_" + g] = torch.from_numpy(z["idx_" + g])
        c[g + "64"] = torch.from_numpy(z[g + "64"])
        c[g + "32"] = torch.from_numpy(z[g + "32"])
        c["scale_" + g] = float(z["scale_" + g])
        c["dist_" + g] = float(z["dist_" + g])
    c["value"] = torch.from_numpy(z["value"])
    return c


def run_vjp(exe, tmp_path, c, feat, grad_output, chunk, want="fpw", options=None, env=None, tag="v"):
    """The backward of one stage -- the map feat [B,C,H,W], the case's points, head and camera -- by emu_fp32's vjp op.
    grad_output: [B,Res,N] or "-" (ones).  -> (dfeat [B,C,H,W], dpoints [B,3,N], [dW_l], [db_l], stdout)"""
    B, C, H, W = feat.shape
    N = c["points"].shape[2]
    inp = dict(feat=feat, rows=c["points"], calib=c["calib"], proj=c["proj"], res=c["chans"][-1], last_op=c["last_op"],
               Ws=c["Ws"], bs=c["bs"], batched=True)
    shapes = [(B, C, H, W), (B, 3, N)] + [tuple(w.shape) for w in c["Ws"]] + [tuple(b.shape) for b in c["bs"]]
    sizes = [int(np.prod(s)) for s in shapes]
    out, r = run(exe, tmp_path, "vjp", B, grad_output, chunk, want, inp=inp, shape=(sum(sizes),),
                 options=dict(widths=",".join(str(x) for x in c["chans"][1:]), **(options or {})), env=env, tag=tag)
    parts = [t.reshape(s) for t, s in zip(out.split(sizes), shapes)]
    L = len(c["Ws"])
    return parts[0], parts[1], parts[2:2 + L], parts[2 + L:], r.stdout


def golden_bar(got_flat, c, g):
    """vjp_bar on a golden's stored components of gradient g (the scale: max|g64| over all components)"""
    got = got_flat[c["idx_" + g]].double()
    ref = c[g + "64"].double()
    scale = c["scale_" + g]
    err = (got - ref).abs() / scale
    worst, frac = err.max().item(), (err <= 2e-5).double().mean().item()
    bar = max(1e-3, 1.1 * c["dist_" + g])
    return worst <= bar and frac >= 0.99, "%s %s: max|err|/max|g| = %.2e (bar %.2e), within 2e-5: %.4f" % (
        c["name"], g, worst, bar, frac)


def head_module(chans, last_op, Ws, bs):
    """a SurfaceClassifier of widths `chans` (skip connections) holding Ws / bs"""
    from monoport_b200.modeling.heads import SurfaceClassifier
    op = {spec.LAST_SIGMOID: nn.Sigmoid(), spec.LAST_TANH: nn.Tanh(), spec.LAST_NONE: None}[last_op]
    h = SurfaceClassifier(chans, 1, False, op)
    h.load_state_dict({**{"filters.%d.weight" % l: W[:, :, None].clone() for l, W in enumerate(Ws)},
                       **{"filters.%d.bias" % l: b.clone() for l, b in enumerate(bs)}})
    return h


def build_vjp_net(chans, last_op, Ws, bs, proj="orthogonal", device="cuda"):
    """a MonoPortNet whose head has widths `chans` and the given weights (on `device`), precision fp32"""
    from monoport_b200.modeling import PIFuNetG
    from monoport_b200.modeling.geometry import perspective
    net = PIFuNetG()
    net.surface_classifier = head_module(chans, last_op, Ws, bs).to(device)
    if proj == "perspective":
        net.projection = perspective
    net.precision = "fp32"
    return net
