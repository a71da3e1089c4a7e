#!/usr/bin/env python
"""Generate tests/golden/bgrad_*.npz by running the UNMODIFIED reference (/root/reference) on CPU: its query() over the batch
of B images of each batch_*.npz case, with `points.requires_grad_()`, differentiated by autograd with respect to the
points, once in fp32 and once in fp64 (head, features, points and calibs all converted).

Run in the build container (the reference tree does not exist on the GPU box):
    python tests/golden/make_batch_grad_golden.py

The inputs are those of tests/golden/make_batch_golden.py, rebuilt from the seeds stored in batch_<case>.npz and checked
against its points and checksums, so the files store only the gradients (and, for the colour case, a seeded grad_output).
N = 1000, 2049 and 515 are ragged against the 16-point tiles of the tensor-core gradient program and the 8- to 32-point
tiles of the exact kernel; the points of every image start with border_points() (on the border, the corners and far
outside).  In g_mixed image 1 has x4 features, above the geometry head's tensor-core limit of 12.  The files are written
with fixed zip timestamps, so a rerun reproduces them byte for byte.
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
from make_golden import border_points, checksum, load_head  # noqa: E402
from make_batch_golden import BATCH_CASES, batch_calib  # noqa: E402
from make_shape_golden import save_npz  # noqa: E402
from grad_cases import query_grad_ref  # noqa: E402

# the seed of the colour case's grad_output [B,3,N]; the geometry cases use ones
GOUT_SEEDS = {"c_rot": 256}


def batch_inputs(c):
    """the batch of make_batch_golden's case c, rebuilt from its seeds and checked against batch_<name>.npz"""
    g = np.load(os.path.join(HERE, "batch_%s.npz" % c["name"]))
    chans = spec.G_CHANNELS if c["net"] == "G" else spec.C_CHANNELS
    Ws, bs = spec.make_weights(chans, c["wseed"])
    feats = [spec.make_feat(chans[0] - 1, c["hw"], c["hw"], fs, sc) for fs, _, sc in c["images"]]
    points = torch.cat([border_points(spec.make_points(c["N"], ps)) for _, ps, _ in c["images"]], 0)
    cals = [batch_calib(c["calib"], b) for b in range(len(c["images"]))]
    calib = torch.cat(cals, 0) if cals[0] is not None else None
    assert np.array_equal(points.numpy(), g["points"]), c["name"]
    assert np.array_equal(calib.numpy() if calib is not None else np.zeros((0,), np.float32), g["calib"]), c["name"]
    np.testing.assert_allclose(np.stack([checksum(w) for w in Ws]), g["w_checksum"], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(np.stack([checksum(f) for f in feats]), g["f_checksum"], rtol=1e-12, atol=1e-12)
    return chans, Ws, bs, torch.cat(feats, 0), points, calib


def reference_batch_grad(ns, c, Ws, bs, feat, points, calib, gout, dtype):
    """the reference's query() (eval, 4 stages of which only the last is used) over the batch, differentiated with respect to
    the points -> (value [B,Res,N], d points [B,3,N])"""
    net = (ns.PIFuNetG() if c["net"] == "G" else ns.PIFuNetC()).eval()
    if c["proj"] == "perspective":
        net.projection = ns.perspective
    load_head(net, Ws, bs)
    net = net.to(dtype)
    f = feat.to(dtype)
    p = points.to(dtype).clone().requires_grad_()
    cal = calib.to(dtype) if calib is not None else None
    decoy = torch.zeros_like(f)
    out = net.query([[decoy], [decoy], [decoy], [f]], p, calibs=cal)
    assert len(out) == 1
    g = torch.ones_like(out[0]) if gout is None else gout.to(dtype)
    (out[0] * g).sum().backward()
    return out[0].detach(), p.grad


def gen_batch_grad(ns):
    for c in BATCH_CASES:
        chans, Ws, bs, feat, points, calib = batch_inputs(c)
        last_op = spec.LAST_SIGMOID if c["net"] == "G" else spec.LAST_TANH
        B, N = points.shape[0], points.shape[2]
        gout = None
        if c["name"] in GOUT_SEEDS:
            gout = torch.randn(B, chans[-1], N, generator=torch.Generator().manual_seed(GOUT_SEEDS[c["name"]]))
        val32, g32 = reference_batch_grad(ns, c, Ws, bs, feat, points, calib, gout, torch.float32)
        _, g64 = reference_batch_grad(ns, c, Ws, bs, feat, points, calib, gout, torch.float64)
        # the differentiable restatement, image by image, against the reference's batch
        for b in range(B):
            cal = calib[b:b + 1] if calib is not None else None
            go = gout[b] if gout is not None else None
            mv, _ = query_grad_ref(feat[b:b + 1], points[b:b + 1], cal, Ws, bs, last_op, c["proj"], grad_output=go)
            _, m64 = query_grad_ref(feat[b:b + 1], points[b:b + 1], cal, Ws, bs, last_op, c["proj"], grad_output=go,
                                    dtype=torch.float64)
            scale = g64[b].abs().max().item()
            e32 = (g32[b].double() - g64[b]).abs()
            print("bgrad %-10s b=%d N=%5d  in-img %.2f  max|g| %.3g  |ref32-ref64|/max: max %.2e, >1e-5: %d   "
                  "|oracle64-ref64|/max %.2e" % (
                      c["name"], b, N, (val32[b, 0] != 0).double().mean().item(), scale, e32.max().item() / scale,
                      int((e32 > 1e-5 * scale).sum()), (m64 - g64[b]).abs().max().item() / scale))
            assert (mv - val32[b]).abs().max().item() < 2e-6
            assert (m64 - g64[b]).abs().max().item() <= 1e-9 * scale
        save_npz(os.path.join(HERE, "bgrad_%s.npz" % c["name"]), value=val32.numpy(), grad32=g32.numpy(),
                 grad64=g64.numpy(), grad_output=(gout.numpy() if gout is not None else np.zeros((0,), np.float32)))


if __name__ == "__main__":
    torch.set_num_threads(8)
    gen_batch_grad(load_reference())
    print("done")
