#!/usr/bin/env python
"""Generate tests/golden/batch_*.npz by running the UNMODIFIED reference (/root/reference) on CPU: its query() over a batch
of B images (features [B,C,H,W], points [B,3,N], calibs [B,4,4] or None), each image with its own map, points and camera.

Run in the build container (the reference tree does not exist on the GPU box):
    python tests/golden/make_batch_golden.py

Like tests/golden/make_golden.py (whose helpers this uses), the large inputs are not stored but regenerated from seeds; each
file stores checksums of the regenerated tensors.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "..", ".."))

from oracle import spec  # noqa: E402
from oracle.ref_loader import load_reference  # noqa: E402
from make_golden import border_points, checksum, load_head  # noqa: E402


BATCH_CASES = [
    # name, net, wseed, per-image (fseed, pseed, fscale), N, calib, projection, feat_hw
    dict(name="g_rot", net="G", wseed=211, images=[(212, 213, 1.0), (214, 215, 1.0), (216, 217, 1.0)], N=1000, calib="rot",
         proj="orthogonal", hw=128),
    dict(name="g_persp", net="G", wseed=221, images=[(222, 223, 1.0), (224, 225, 1.0)], N=2049, calib="persp",
         proj="perspective", hw=128),
    dict(name="g_nocalib", net="G", wseed=231, images=[(232, 233, 1.0), (234, 235, 1.0)], N=1000, calib="none",
         proj="orthogonal", hw=32),
    # image 1: features x4 (max |feature| ~ 21, above the geometry head's tensor-core limit of 12)
    dict(name="g_mixed", net="G", wseed=241, images=[(242, 243, 1.0), (244, 245, 4.0), (246, 247, 1.0)], N=1000, calib="rot",
         proj="orthogonal", hw=128),
    dict(name="c_rot", net="C", wseed=251, images=[(252, 253, 1.0), (254, 255, 1.0)], N=515, calib="rot", proj="orthogonal",
         hw=128),
]


def batch_calib(kind, b):
    """A different camera per image of a batch."""
    if kind == "rot":
        return spec.scene_calib(20.0 + 15.0 * b, 33.0 - 40.0 * b)
    if kind == "persp":
        c = spec.scene_calib(10.0 + 10.0 * b, -15.0 + 20.0 * b).clone()
        c[0, 2, 3] = 3.0
        c[0, :2, :] *= 2.5
        return c
    if kind == "none":
        return None
    raise ValueError(kind)


@torch.no_grad()
def gen_batch_query(ns):
    """tests/golden/batch_*.npz: the reference's query() on a batch of B images (features [B,C,H,W], points [B,3,N], calibs
    [B,4,4] or None) -- one call, each image with its own map, points and camera."""
    for c in BATCH_CASES:
        chans = spec.G_CHANNELS if c["net"] == "G" else spec.C_CHANNELS
        last_op = spec.LAST_SIGMOID if c["net"] == "G" else spec.LAST_TANH
        net = (ns.PIFuNetG() if c["net"] == "G" else ns.PIFuNetC()).eval()
        if c["proj"] == "perspective":
            net.projection = ns.perspective
        Ws, bs = spec.make_weights(chans, c["wseed"])
        load_head(net, Ws, bs)
        C = chans[0] - 1
        feats = [spec.make_feat(C, c["hw"], c["hw"], fs, sc) for fs, _, sc in c["images"]]
        pts = [border_points(spec.make_points(c["N"], ps)) for _, ps, _ in c["images"]]
        cals = [batch_calib(c["calib"], b) for b in range(len(c["images"]))]
        feat = torch.cat(feats, 0)
        points = torch.cat(pts, 0)
        calib = torch.cat(cals, 0) if cals[0] is not None else None
        decoy = torch.zeros_like(feat)
        out = net.query([[decoy], [decoy], [decoy], [feat]], points, calibs=calib)
        assert len(out) == 1
        ref = out[0].numpy()
        err = 0.0
        for b in range(len(feats)):
            mine = spec.query_ref(feats[b], pts[b], cals[b], Ws, bs, last_op, c["proj"]).numpy()
            err = max(err, np.abs(ref[b] - mine).max())
        print("batch %-10s B=%d N=%5d  |oracle per image - ref| = %.2e" % (c["name"], len(feats), c["N"], err))
        assert err < 2e-6
        np.savez_compressed(
            os.path.join(HERE, "batch_%s.npz" % c["name"]),
            points=points.numpy(), calib=(calib.numpy() if calib is not None else np.zeros((0,), np.float32)),
            expected=ref, net=c["net"], wseed=c["wseed"], fseeds=np.array([i[0] for i in c["images"]]),
            pseeds=np.array([i[1] for i in c["images"]]), fscales=np.array([i[2] for i in c["images"]]), hw=c["hw"],
            proj=c["proj"], w_checksum=np.stack([checksum(w) for w in Ws]), f_checksum=np.stack([checksum(f) for f in feats]))


if __name__ == "__main__":
    torch.set_num_threads(8)
    gen_batch_query(load_reference())
    print("done")
