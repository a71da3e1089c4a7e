"""The head goldens (tests/golden/head_*.npz, written by tests/golden/make_head_golden.py: the reference's query() and its
point gradient with heads other than the two shipped ones) and the regeneration of the seeded inputs they do not store."""
import os

import numpy as np
import torch

from oracle import spec
from helpers import GOLDEN, checksum
from shape_cases import _names

SHIPPED = {"G": spec.G_CHANNELS, "C": spec.C_CHANNELS}
MAX_SMEM_OPTIN = 232448          # the H100's shared-memory opt-in per block, which the CPU model reports


def head_cases():
    return [n for n in _names("head_") if not n.startswith("grad_")]


def head_grad_cases():
    return _names("head_grad_")


def head_widths(name):
    """filter_channels of a head golden, without regenerating its inputs"""
    return [int(x) for x in np.load(os.path.join(GOLDEN, "head_%s.npz" % name))["chans"]]


def shipped_widths(chans):
    """"G" / "C" when `chans` are the widths of a shipped head (the tensor-core programs' widths), else None"""
    return next((k for k, v in SHIPPED.items() if list(chans) == v), None)


def fp32_tile(chans, max_smem=MAX_SMEM_OPTIN, grad=False):
    """The tile size P of the exact kernels for a head, from their shared-memory footprint: [c0 + ping + pong][P] floats of
    activations (ping / pong: the widest even / odd hidden layer), [8][P] of point metadata and, for the gradient, one sign
    word per 32 hidden channels and [Res][P] floats; the largest P in 32, 16, 8 that fits with 2 KB to spare.  None: refused."""
    L = len(chans) - 1
    hidden = chans[1:L]
    ping = max(hidden[0::2], default=0)
    pong = max(hidden[1::2], default=0)
    for P in (32, 16, 8):
        need = (chans[0] + ping + pong) * P * 4 + P * 8 * 4
        if grad:
            need += sum((c + 31) // 32 for c in hidden) * P * 4 + chans[-1] * P * 4
        if need + 2048 <= max_smem:
            return P
    return None


def _load(prefix, name):
    g = np.load(os.path.join(GOLDEN, "%s%s.npz" % (prefix, name)))
    chans = [int(x) for x in g["chans"]]
    Ws, bs = spec.make_weights(chans, int(g["wseed"]))
    amax = float(g["amax"])
    feat = spec.make_feat(chans[0] - 1, int(g["H"]), int(g["W"]), int(g["fseed"]))
    if not np.isnan(amax):
        feat = feat * (amax / feat.abs().max().item())
    # RNG drift must fail loudly, not as a parity error
    np.testing.assert_allclose(np.concatenate([checksum(w) for w in Ws]), g["w_checksum"], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(checksum(feat), g["f_checksum"], rtol=1e-12, atol=1e-12)
    return g, dict(name=name, chans=chans, last_op=int(g["last_op"]), Ws=Ws, bs=bs, feat=feat, H=int(g["H"]), W=int(g["W"]),
                   proj=str(g["proj"]), amax=None if np.isnan(amax) else amax, net=shipped_widths(chans),
                   calib=torch.from_numpy(g["calib"]) if g["calib"].size else None, points=torch.from_numpy(g["points"]))


def load_head_case(name):
    """-> dict(chans, last_op, Ws, bs, feat [1,C,H,W], points [1,3,N], calib [1,4,4]|None, proj, expected / expected64
    [Res,N], amax (the map's largest |feature| when the golden sets it), net ("G"/"C" on the shipped widths, else None))"""
    g, c = _load("head_", name)
    return dict(c, expected=torch.from_numpy(g["expected"]), expected64=torch.from_numpy(g["expected64"]))


def load_head_grad_case(name):
    """-> dict(..., value [Res,N], grad32 / grad64 [3,N]: the reference's fp32 / fp64 autograd gradient of sum(query()))"""
    g, c = _load("head_grad_", name)
    return dict(c, value=torch.from_numpy(g["value"]), grad32=torch.from_numpy(g["grad32"]),
                grad64=torch.from_numpy(g["grad64"]), grad_output=None)


def build_head_net(c, device="cuda", no_residual=False):
    """monoport_b200 MonoPortNet (eval) whose head is SurfaceClassifier(c["chans"], 1, no_residual, last_op) with the case's
    weights (no_residual=True: a head of the same widths without the skip inputs, seeded like the case)"""
    import torch.nn as nn
    from monoport_b200.modeling import PIFuNetG
    from monoport_b200.modeling.geometry import perspective
    from monoport_b200.modeling.heads import SurfaceClassifier
    net = PIFuNetG()
    last = {spec.LAST_SIGMOID: nn.Sigmoid(), spec.LAST_TANH: nn.Tanh(), spec.LAST_NONE: None}[c["last_op"]]
    net.surface_classifier = SurfaceClassifier(c["chans"], 1, no_residual, last)
    if not no_residual:
        sd = {}
        for l, (W, b) in enumerate(zip(c["Ws"], c["bs"])):
            sd["filters.%d.weight" % l] = W[:, :, None].clone()
            sd["filters.%d.bias" % l] = b.clone()
        net.surface_classifier.load_state_dict(sd)
    if c["proj"] == "perspective":
        net.projection = perspective
    net.surface_classifier.to(device)
    return net.eval()
