"""The map-shape goldens (tests/golden/shape_*.npz, written by tests/golden/make_shape_golden.py: the reference's query(), its
point gradient and its batched query() on feature maps that are not square, whose texel count is not a multiple of 128, that
sit at or above 65536 texels, or that have an axis of length 1) and the regeneration of the seeded inputs they do not store."""
import glob
import os

import numpy as np
import torch

from oracle import spec
from helpers import GOLDEN, checksum

TC_TEXEL_LIMIT = 65536          # the tensor-core program's largest map (texel offsets travel as 16-bit pairs)


def _names(prefix):
    return sorted(os.path.basename(p)[len(prefix):-4] for p in glob.glob(os.path.join(GOLDEN, prefix + "*.npz")))


def shape_cases():
    """single-map query goldens"""
    return [n for n in _names("shape_") if not n.startswith(("grad_", "batch_"))]


def shape_grad_cases():
    return _names("shape_grad_")


def shape_batch_cases():
    return _names("shape_batch_")


def _head(g):
    net = str(g["net"])
    chans = spec.G_CHANNELS if net == "G" else spec.C_CHANNELS
    Ws, bs = spec.make_weights(chans, int(g["wseed"]))
    # RNG drift must fail loudly, not as a parity error
    np.testing.assert_allclose(np.stack([checksum(w) for w in Ws]), g["w_checksum"], rtol=1e-12, atol=1e-12)
    return dict(net=net, chans=chans, Ws=Ws, bs=bs, last_op=spec.LAST_SIGMOID if net == "G" else spec.LAST_TANH,
                proj=str(g["proj"]), H=int(g["H"]), W=int(g["W"]),
                calib=torch.from_numpy(g["calib"]) if g["calib"].size else None, points=torch.from_numpy(g["points"]))


def _feat(g, chans, fseed):
    return spec.make_feat(chans[0] - 1, int(g["H"]), int(g["W"]), int(fseed))


def load_shape_case(name):
    """-> dict(points [1,3,N], calib [1,4,4]|None, expected [Res,N], feat [1,C,H,W], H, W, Ws, bs, last_op, proj, net)"""
    g = np.load(os.path.join(GOLDEN, "shape_%s.npz" % name))
    c = _head(g)
    c["feat"] = _feat(g, c["chans"], g["fseed"])
    np.testing.assert_allclose(checksum(c["feat"]), g["f_checksum"], rtol=1e-12, atol=1e-12)
    return dict(c, name=name, expected=torch.from_numpy(g["expected"]), expected64=torch.from_numpy(g["expected64"]))


def within_fp32_bar(got, c, bar=2e-5):
    """The bar of the exact fp32 kernel: within `bar` of the reference's fp32 output.  Where the reference's own fp32 rounding
    is already farther than `bar` from its float64 result (the colour head's 1537-wide layers reach 3.6e-5 on c_over), the
    golden cannot resolve that bar: the kernel must then be no farther from the float64 result than the reference's fp32
    output is, within 10 %.  -> (ok, message)"""
    got = got.double()
    err = (got - c["expected"].double()).abs().max().item()
    own = (c["expected"].double() - c["expected64"]).abs().max().item()
    if own <= bar:
        return err <= bar, "max|got - ref32| = %.2e" % err
    e64 = (got - c["expected64"]).abs().max().item()
    return e64 <= 1.1 * own, "max|got - ref64| = %.2e, max|ref32 - ref64| = %.2e" % (e64, own)


def load_shape_grad_case(name):
    """-> dict(points [1,3,N], calib, value [Res,N], grad32 / grad64 [3,N], grad_output None, feat, H, W, Ws, bs, ...) -- the
    layout of tests/grad_cases.load_grad_case"""
    g = np.load(os.path.join(GOLDEN, "shape_grad_%s.npz" % name))
    c = _head(g)
    c["feat"] = _feat(g, c["chans"], g["fseed"])
    np.testing.assert_allclose(checksum(c["feat"]), g["f_checksum"], rtol=1e-12, atol=1e-12)
    return dict(c, name=name, value=torch.from_numpy(g["value"]), grad32=torch.from_numpy(g["grad32"]),
                grad64=torch.from_numpy(g["grad64"]), grad_output=None)


def load_shape_batch_case(name):
    """-> dict(points [B,3,N], calib [B,4,4]|None, expected [B,Res,N], feat [B,C,H,W], B, H, W, Ws, bs, ...) -- the layout of
    tests/batch_cases.load_batch_case"""
    g = np.load(os.path.join(GOLDEN, "shape_batch_%s.npz" % name))
    c = _head(g)
    feats = [_feat(g, c["chans"], fs) for fs in g["fseeds"]]
    np.testing.assert_allclose(np.stack([checksum(f) for f in feats]), g["f_checksum"], rtol=1e-12, atol=1e-12)
    return dict(c, name=name, feat=torch.cat(feats, 0), B=len(feats), expected=torch.from_numpy(g["expected"]))
