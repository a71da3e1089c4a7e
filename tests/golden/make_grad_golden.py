#!/usr/bin/env python
"""Generate tests/golden/grad_*.npz by running the UNMODIFIED reference (/root/reference) on CPU: its query() with
`points.requires_grad_()`, differentiated by autograd, once in fp32 and once in fp64 (head, features, points and calib all
converted).

Run in the build container (the reference tree does not exist on the GPU box):
    python tests/golden/make_grad_golden.py

Like tests/golden/make_golden.py (whose helpers this uses), the large inputs are not stored but regenerated from seeds; each
file stores checksums of the regenerated tensors.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, os.path.join(HERE, "..", ".."))

from oracle import spec  # noqa: E402
from oracle.ref_loader import load_reference  # noqa: E402
from make_golden import border_points, checksum, load_head, make_calib  # noqa: E402
from grad_cases import query_grad_ref  # noqa: E402


GRAD_CASES = [
    # name, net, wseed, fseed, pseed, N, calib, projection, feat_scale, feat_hw, grad_output seed (None = ones)
    dict(name="g_rot", net="G", wseed=3, fseed=4, pseed=5, N=2000, calib="rot33", proj="orthogonal", fscale=1.0, hw=128, gseed=None),
    dict(name="g_persp", net="G", wseed=301, fseed=302, pseed=303, N=1000, calib="persp", proj="perspective", fscale=1.0, hw=128,
         gseed=None),
    dict(name="g_nocalib", net="G", wseed=311, fseed=312, pseed=313, N=1000, calib="none", proj="orthogonal", fscale=1.0, hw=32,
         gseed=None),
    dict(name="g_bigfeat", net="G", wseed=321, fseed=322, pseed=323, N=1000, calib="rot33", proj="orthogonal", fscale=4.0, hw=128,
         gseed=None),
    dict(name="c_rot", net="C", wseed=331, fseed=332, pseed=333, N=515, calib="rot33", proj="orthogonal", fscale=1.0, hw=128,
         gseed=334),
]


def reference_grad(ns, c, Ws, bs, feat, pts, calib, gout, dtype):
    """the reference's query() (eval, 4 stages of which only the last is used) differentiated with respect to the points"""
    net = (ns.PIFuNetG() if c["net"] == "G" else ns.PIFuNetC()).eval()
    if c["proj"] == "perspective":
        net.projection = ns.perspective
    load_head(net, Ws, bs)
    net = net.to(dtype)
    f = feat.to(dtype)
    p = pts.to(dtype).clone().requires_grad_()
    cal = calib.to(dtype) if calib is not None else None
    decoy = torch.zeros_like(f)
    out = net.query([[decoy], [decoy], [decoy], [f]], p, calibs=cal)
    assert len(out) == 1
    g = torch.ones_like(out[0]) if gout is None else gout[None].to(dtype)
    (out[0] * g).sum().backward()
    return out[0][0].detach(), p.grad[0]


def gen_grad(ns):
    for c in GRAD_CASES:
        chans = spec.G_CHANNELS if c["net"] == "G" else spec.C_CHANNELS
        last_op = spec.LAST_SIGMOID if c["net"] == "G" else spec.LAST_TANH
        Ws, bs = spec.make_weights(chans, c["wseed"])
        feat = spec.make_feat(chans[0] - 1, c["hw"], c["hw"], c["fseed"], c["fscale"])
        pts = border_points(spec.make_points(c["N"], c["pseed"]))
        calib = make_calib(c["calib"])
        gout = None
        if c["gseed"] is not None:
            gout = torch.randn(chans[-1], c["N"], generator=torch.Generator().manual_seed(c["gseed"]))
        val32, g32 = reference_grad(ns, c, Ws, bs, feat, pts, calib, gout, torch.float32)
        _, g64 = reference_grad(ns, c, Ws, bs, feat, pts, calib, gout, torch.float64)
        # the differentiable restatement against the reference, in both precisions
        mv, m32 = query_grad_ref(feat, pts, calib, Ws, bs, last_op, c["proj"], grad_output=gout)
        _, m64 = query_grad_ref(feat, pts, calib, Ws, bs, last_op, c["proj"], grad_output=gout, dtype=torch.float64)
        scale = g64.abs().max().item()
        e32 = (g32.double() - g64).abs()
        print("grad %-10s N=%5d  in-img %.2f  max|g| %.3g  |ref32-ref64|/max: max %.2e, >1e-5: %d, >1e-4: %d, >1e-3: %d   "
              "|oracle64-ref64|/max %.2e  |oracle32-ref32|/max %.2e" % (
                  c["name"], c["N"], (val32[0] != 0).double().mean().item(), scale, e32.max().item() / scale,
                  int((e32 > 1e-5 * scale).sum()), int((e32 > 1e-4 * scale).sum()), int((e32 > 1e-3 * scale).sum()),
                  (m64 - g64).abs().max().item() / scale, (m32 - g32).abs().max().item() / scale))
        assert (mv - val32).abs().max().item() < 2e-6
        assert (m64 - g64).abs().max().item() <= 1e-9 * scale
        np.savez_compressed(
            os.path.join(HERE, "grad_%s.npz" % c["name"]),
            points=pts.numpy(), calib=(calib.numpy() if calib is not None else np.zeros((0,), np.float32)),
            grad_output=(gout.numpy() if gout is not None else np.zeros((0,), np.float32)),
            value=val32.numpy(), grad32=g32.numpy(), grad64=g64.numpy(), net=c["net"], wseed=c["wseed"], fseed=c["fseed"],
            fscale=c["fscale"], hw=c["hw"], proj=c["proj"], w_checksum=np.stack([checksum(w) for w in Ws]),
            f_checksum=checksum(feat))


if __name__ == "__main__":
    torch.set_num_threads(8)
    gen_grad(load_reference())
    print("done")
