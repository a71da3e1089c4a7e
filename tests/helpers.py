"""Shared test helpers: golden loading + regeneration of the seeded inputs the goldens do not store."""
import glob
import os

import numpy as np
import torch

from oracle import spec

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def checksum(t):
    t = t.double().reshape(-1)
    w = torch.arange(1, t.numel() + 1, dtype=torch.float64) % 997
    return np.array([t.sum().item(), (t * w).sum().item(), t.abs().max().item()])


def query_cases():
    return sorted(os.path.basename(p)[len("query_"):-4] for p in glob.glob(os.path.join(GOLDEN, "query_*.npz")))


def load_query_case(name):
    """-> dict(points [1,3,N], calib [1,4,4]|None, expected [Res,N], Ws, bs, feat, last_op, proj, net)"""
    g = np.load(os.path.join(GOLDEN, "query_%s.npz" % name))
    net = str(g["net"])
    chans = spec.G_CHANNELS if net == "G" else spec.C_CHANNELS
    Ws, bs = spec.make_weights(chans, int(g["wseed"]))
    feat = spec.make_feat(chans[0] - 1, int(g["hw"]), int(g["hw"]), int(g["fseed"]), float(g["fscale"]))
    # the goldens store checksums of the regenerated inputs: RNG drift must fail loudly, not as a parity error
    np.testing.assert_allclose(np.stack([checksum(w) for w in Ws]), g["w_checksum"], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(checksum(feat), g["f_checksum"], rtol=1e-12, atol=1e-12)
    calib = torch.from_numpy(g["calib"]) if g["calib"].size else None
    return dict(name=name, net=net, points=torch.from_numpy(g["points"]), calib=calib,
                expected=torch.from_numpy(g["expected"]), Ws=Ws, bs=bs, feat=feat, chans=chans,
                last_op=spec.LAST_SIGMOID if net == "G" else spec.LAST_TANH, proj=str(g["proj"]))


def build_net(case_or_net, Ws=None, bs=None, device="cuda", proj="orthogonal"):
    """monoport_b200 MonoPortNet (eval) with the head weights of a golden case loaded."""
    from monoport_b200.modeling import PIFuNetG, PIFuNetC
    from monoport_b200.modeling.geometry import perspective
    if isinstance(case_or_net, dict):
        net_kind, Ws, bs, proj = case_or_net["net"], case_or_net["Ws"], case_or_net["bs"], case_or_net["proj"]
    else:
        net_kind = case_or_net
    with torch.device("meta"):
        pass
    net = (PIFuNetG() if net_kind == "G" else PIFuNetC())
    sd = {}
    for l, (W, b) in enumerate(zip(Ws, bs)):
        sd["filters.%d.weight" % l] = W[:, :, None].clone()
        sd["filters.%d.bias" % l] = b.clone()
    net.surface_classifier.load_state_dict(sd)
    if proj == "perspective":
        net.projection = perspective
    net.surface_classifier.to(device)
    return net.eval()


def lookup_query(field, b_min=(-1, -1, -1), b_max=(1, 1, 1)):
    """query_func that reads a dense [R,R,R] field at the node nearest to each world point of the box [b_min, b_max]
    (bit-exact on CPU and GPU: pure gather).  The node is recovered in float64 from level_points' convention
    p = (c + 0.5) / R * (b_max - b_min) + b_min.  Returns (fn_oracle(points[N,3])->[N], fn_engine(points=[1,N,3])->[1,1,N])."""
    R = field.shape[0]
    lo = torch.tensor(b_min, dtype=torch.float64)
    ext = torch.tensor(b_max, dtype=torch.float64) - lo

    def idx(p):
        i = ((p.double() - lo.to(p.device)) / ext.to(p.device) * R - 0.5).round().long().clamp(0, R - 1)
        return i[..., 2], i[..., 1], i[..., 0]

    def fn_oracle(p):
        z, y, x = idx(p)
        return field[z, y, x]

    dev_field = {}

    def fn_engine(points, **kw):
        f = dev_field.get(points.device)
        if f is None:
            f = dev_field[points.device] = field.to(points.device)
        z, y, x = idx(points[0])
        return f[z, y, x].view(1, 1, -1)

    return fn_oracle, fn_engine
