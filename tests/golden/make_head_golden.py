#!/usr/bin/env python
"""Generate tests/golden/head_*.npz by running the UNMODIFIED reference (/root/reference) on CPU with heads other than the
two shipped ones: the reference's SurfaceClassifier(filter_channels, 1, no_residual=False, last_op) installed in its
MonoPortNet, each head chosen for an edge of the exact kernels (tile size, widths that are not multiples of 4 or 32, one
layer, eight layers, outputs other than 1 or 3, no last op) or, on the shipped widths, for a last op the shipped heads do
not use (the tensor-core programs' feature limit per last op).

Run in the build container (the reference tree does not exist on the GPU box):
    python tests/golden/make_head_golden.py

Like tests/golden/make_shape_golden.py (whose helpers this uses), the large inputs are not stored but regenerated from seeds;
each file stores checksums of the regenerated tensors, and is written with fixed zip timestamps, so a rerun reproduces it
byte for byte.

Two kinds of file:
  head_<case>.npz       the reference's query() (points, calib, expected; expected64: the same in float64)
  head_grad_<case>.npz  its point gradient by autograd, in fp32 and fp64 (as tests/golden/make_grad_golden.py)
The points are border_points() and then uniform ones.  A case with `amax` scales its seeded map to that largest |feature|.
"""
import os
import sys

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, os.path.join(HERE, "..", ".."))

from oracle import spec  # noqa: E402
from oracle.ref_loader import load_reference  # noqa: E402
from make_golden import border_points, checksum, load_head, make_calib  # noqa: E402
from make_shape_golden import save_npz  # noqa: E402
from grad_cases import query_grad_ref  # noqa: E402

G, C = spec.G_CHANNELS, spec.C_CHANNELS
S, T, NONE = spec.LAST_SIGMOID, spec.LAST_TANH, spec.LAST_NONE

HEAD_CASES = [
    # name, filter_channels, last op, map H x W, seeds, points, calib, projection, gradient golden, max |feature| (None: as
    # seeded)
    dict(name="narrow", chans=[33, 64, 48, 1], last_op=S, H=9, W=13, wseed=601, fseed=602, pseed=603, N=520, calib="rot33",
         proj="orthogonal", grad=True, amax=None),
    dict(name="odd", chans=[20, 300, 77, 130, 5, 2], last_op=NONE, H=11, W=6, wseed=611, fseed=612, pseed=613, N=520,
         calib="persp", proj="perspective", grad=True, amax=None),
    dict(name="single", chans=[65, 3], last_op=T, H=7, W=10, wseed=621, fseed=622, pseed=623, N=520, calib="none",
         proj="orthogonal", grad=True, amax=None),
    dict(name="deep", chans=[40, 32, 32, 33, 31, 64, 16, 8, 1], last_op=S, H=12, W=5, wseed=631, fseed=632, pseed=633, N=520,
         calib="rot33", proj="orthogonal", grad=True, amax=None),
    dict(name="g128", chans=[129, 1024, 512, 256, 128, 1], last_op=S, H=16, W=24, wseed=641, fseed=642, pseed=643, N=520,
         calib="rot33", proj="orthogonal", grad=True, amax=None),
    dict(name="g_res3", chans=[257, 1024, 512, 256, 128, 3], last_op=T, H=20, W=14, wseed=651, fseed=652, pseed=653, N=520,
         calib="rot33", proj="orthogonal", grad=True, amax=None),
    dict(name="p32_full", chans=[1025, 512, 255, 1], last_op=S, H=6, W=5, wseed=661, fseed=662, pseed=663, N=520,
         calib="rot33", proj="orthogonal", grad=True, amax=None),
    dict(name="p8_full", chans=[1025, 4096, 2071, 1], last_op=S, H=5, W=4, wseed=671, fseed=672, pseed=673, N=72,
         calib="rot33", proj="orthogonal", grad=False, amax=None),
    # the gradient's tile 8 (the query's too), with several outer passes of the transposed layers
    dict(name="p8", chans=[65, 3000, 600, 1], last_op=S, H=8, W=11, wseed=721, fseed=722, pseed=723, N=120,
         calib="rot33", proj="orthogonal", grad=True, amax=None),
    # the shipped widths with the other last ops, the map at 0.99 x the head's default feature limit
    dict(name="sdf", chans=G, last_op=NONE, H=48, W=40, wseed=681, fseed=682, pseed=683, N=520, calib="rot33",
         proj="orthogonal", grad=False, amax=0.99 * 3.0),
    dict(name="g_tanh", chans=G, last_op=T, H=48, W=40, wseed=691, fseed=692, pseed=693, N=520, calib="rot33",
         proj="orthogonal", grad=False, amax=0.99 * 3.0),
    dict(name="csig", chans=C, last_op=S, H=40, W=32, wseed=701, fseed=702, pseed=703, N=520, calib="rot33",
         proj="orthogonal", grad=False, amax=0.99 * 12.0),
    dict(name="c_none", chans=C, last_op=NONE, H=40, W=32, wseed=711, fseed=712, pseed=713, N=520, calib="rot33",
         proj="orthogonal", grad=False, amax=0.99 * 4.0),
]


def case_feat(c):
    feat = spec.make_feat(c["chans"][0] - 1, c["H"], c["W"], c["fseed"])
    if c["amax"] is not None:
        feat = feat * (c["amax"] / feat.abs().max().item())
    return feat


def reference_net(ns, c, Ws, bs, dtype=torch.float32):
    """the reference's MonoPortNet with SurfaceClassifier(chans, 1, False, last_op) as its head"""
    net = ns.PIFuNetG().eval()
    last = {S: nn.Sigmoid(), T: nn.Tanh(), NONE: None}[c["last_op"]]
    net.surface_classifier = ns.SurfaceClassifier(c["chans"], 1, False, last)
    if c["proj"] == "perspective":
        net.projection = ns.perspective
    load_head(net, Ws, bs)
    return net.eval().to(dtype)


def reference_query(ns, c, Ws, bs, feat, pts, calib, dtype):
    net = reference_net(ns, c, Ws, bs, dtype)
    f = feat.to(dtype)
    decoy = torch.zeros_like(f)
    with torch.no_grad():
        out = net.query([[decoy], [decoy], [decoy], [f]], pts.to(dtype), calibs=calib.to(dtype) if calib is not None else None)
    assert len(out) == 1
    return out[0][0]


def reference_grad(ns, c, Ws, bs, feat, pts, calib, dtype):
    """the reference's query() differentiated with respect to the points (grad_output = ones)"""
    net = reference_net(ns, c, Ws, bs, dtype)
    f = feat.to(dtype)
    p = pts.to(dtype).clone().requires_grad_()
    decoy = torch.zeros_like(f)
    out = net.query([[decoy], [decoy], [decoy], [f]], p, calibs=calib.to(dtype) if calib is not None else None)
    out[0].sum().backward()
    return out[0][0].detach(), p.grad[0]


def common(c, Ws, feat, pts, calib):
    return dict(points=pts.numpy(), calib=(calib.numpy() if calib is not None else np.zeros((0,), np.float32)),
                chans=np.array(c["chans"], np.int32), last_op=c["last_op"], wseed=c["wseed"], fseed=c["fseed"], H=c["H"],
                W=c["W"], proj=c["proj"], amax=np.float64(np.nan if c["amax"] is None else c["amax"]),
                w_checksum=np.concatenate([checksum(w) for w in Ws]), f_checksum=checksum(feat))


def gen_heads(ns):
    for c in HEAD_CASES:
        Ws, bs = spec.make_weights(c["chans"], c["wseed"])
        feat = case_feat(c)
        calib = make_calib(c["calib"])
        pts = border_points(spec.make_points(c["N"], c["pseed"]))
        ref = reference_query(ns, c, Ws, bs, feat, pts, calib, torch.float32)
        ref64 = reference_query(ns, c, Ws, bs, feat, pts, calib, torch.float64)
        mine = spec.query_ref(feat, pts, calib, Ws, bs, c["last_op"], c["proj"])
        err = (ref - mine).abs().max().item()
        print("head %-9s %-36s N=%4d  in-img %.2f  |oracle-ref| = %.2e  |ref32-ref64| = %.2e" % (
            c["name"], c["chans"], c["N"], (ref[0] != 0).double().mean().item(), err,
            (ref.double() - ref64).abs().max().item()))
        assert err < 2e-6
        save_npz(os.path.join(HERE, "head_%s.npz" % c["name"]), kind="query", expected=ref.numpy(), expected64=ref64.numpy(),
                 **common(c, Ws, feat, pts, calib))
        if not c["grad"]:
            continue
        val32, g32 = reference_grad(ns, c, Ws, bs, feat, pts, calib, torch.float32)
        _, g64 = reference_grad(ns, c, Ws, bs, feat, pts, calib, torch.float64)
        mv, m32 = query_grad_ref(feat, pts, calib, Ws, bs, c["last_op"], c["proj"])
        _, m64 = query_grad_ref(feat, pts, calib, Ws, bs, c["last_op"], c["proj"], dtype=torch.float64)
        scale = g64.abs().max().item()
        print("     grad  max|g| %.3g  |ref32-ref64|/max %.2e  |oracle64-ref64|/max %.2e  |oracle32-ref32|/max %.2e" % (
            scale, (g32.double() - g64).abs().max().item() / scale, (m64 - g64).abs().max().item() / scale,
            (m32 - g32).abs().max().item() / scale))
        assert (mv - val32).abs().max().item() < 2e-6
        assert (m64 - g64).abs().max().item() <= 1e-9 * scale
        save_npz(os.path.join(HERE, "head_grad_%s.npz" % c["name"]), kind="grad", value=val32.numpy(), grad32=g32.numpy(),
                 grad64=g64.numpy(), **common(c, Ws, feat, pts, calib))


if __name__ == "__main__":
    torch.set_num_threads(8)
    gen_heads(load_reference())
    print("done")
