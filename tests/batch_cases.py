"""The batched query goldens (tests/golden/batch_*.npz, the reference's query() over B images) and the regeneration of the
seeded inputs they do not store."""
import glob
import os

import numpy as np
import torch

from oracle import spec
from helpers import GOLDEN, checksum


def batch_cases():
    return sorted(os.path.basename(p)[len("batch_"):-4] for p in glob.glob(os.path.join(GOLDEN, "batch_*.npz")))


def load_batch_case(name):
    """-> dict(points [B,3,N], calib [B,4,4]|None, expected [B,Res,N], feat [B,C,H,W], Ws, bs, last_op, proj, net, B)"""
    g = np.load(os.path.join(GOLDEN, "batch_%s.npz" % name))
    net = str(g["net"])
    chans = spec.G_CHANNELS if net == "G" else spec.C_CHANNELS
    Ws, bs = spec.make_weights(chans, int(g["wseed"]))
    hw = int(g["hw"])
    feats = [spec.make_feat(chans[0] - 1, hw, hw, int(fs), float(sc)) for fs, sc in zip(g["fseeds"], g["fscales"])]
    # RNG drift must fail loudly, not as a parity error
    np.testing.assert_allclose(np.stack([checksum(w) for w in Ws]), g["w_checksum"], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(np.stack([checksum(f) for f in feats]), g["f_checksum"], rtol=1e-12, atol=1e-12)
    calib = torch.from_numpy(g["calib"]) if g["calib"].size else None
    return dict(name=name, net=net, points=torch.from_numpy(g["points"]), calib=calib, expected=torch.from_numpy(g["expected"]),
                Ws=Ws, bs=bs, feat=torch.cat(feats, 0), chans=chans, B=len(feats), fscales=[float(s) for s in g["fscales"]],
                last_op=spec.LAST_SIGMOID if net == "G" else spec.LAST_TANH, proj=str(g["proj"]))
