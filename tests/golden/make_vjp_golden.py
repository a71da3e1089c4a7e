#!/usr/bin/env python
"""Generate tests/golden/vjp_*.npz by running the UNMODIFIED reference (/root/reference) on CPU: its train-mode query() (every
stage evaluated, MonoPortNet.py:63-91) with the feature maps, the points and the head's parameters requiring grad,
differentiated by autograd, once in fp32 and once in fp64 (head, features, points and calib all converted).

Run in the build container (the reference tree does not exist on the GPU box):
    python tests/golden/make_vjp_golden.py

The inputs are regenerated from seeds (tests/vjp_cases.py: make_case_inputs).  A weight gradient of the geometry head has
1.3 M components, so each file stores, per gradient (d features of all stages, d points, d weights and d biases of all
layers), a seeded sample of 4096 components (all of them for smaller gradients) in fp64 and fp32, the largest |fp64|
component over all of them, and the largest distance of the reference's fp32 gradient from its fp64 one over all of them
(printed, and the bar's floor where it exceeds 1e-3).  The zip entries carry a fixed timestamp: a rerun is byte-identical.
"""
import io
import os
import sys
import zipfile

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, os.path.join(HERE, "..", ".."))

from oracle import spec  # noqa: E402
from oracle.ref_loader import load_reference  # noqa: E402
from vjp_cases import GRAD_NAMES, flat, make_case_inputs, query_vjp_ref, sample_index  # noqa: E402

NARROW = [33, 64, 48, 1]          # tests/golden/head_grad_narrow.npz's widths (head_cases.py)

VJP_CASES = [
    # chans, last_op, B images, S stages, N points per image, H x W map, camera, grad_output seed (-1: ones)
    dict(name="g_b1_rot", chans=spec.G_CHANNELS, last_op="sigmoid", B=1, S=1, N=301, H=32, W=32, calib="rot", gseed=-1,
         wseed=401, fseed=402, pseed=403),
    dict(name="g_b3_s4_persp", chans=spec.G_CHANNELS, last_op="sigmoid", B=3, S=4, N=97, H=16, W=16, calib="persp", gseed=-1,
         wseed=411, fseed=412, pseed=413),
    dict(name="g_b1_nocalib_nonsquare", chans=spec.G_CHANNELS, last_op="sigmoid", B=1, S=1, N=150, H=24, W=40, calib="none",
         gseed=-1, wseed=421, fseed=422, pseed=423),
    dict(name="c_b3_rot", chans=spec.C_CHANNELS, last_op="tanh", B=3, S=1, N=71, H=16, W=16, calib="rot", gseed=434,
         wseed=431, fseed=432, pseed=433),
    dict(name="c_b1_s4_rot", chans=spec.C_CHANNELS, last_op="tanh", B=1, S=4, N=40, H=16, W=16, calib="rot", gseed=444,
         wseed=441, fseed=442, pseed=443),
    dict(name="narrow_b3_persp", chans=NARROW, last_op="sigmoid", B=3, S=2, N=211, H=20, W=12, calib="persp", gseed=454,
         wseed=451, fseed=452, pseed=453),
]


def reference_vjp(ns, c, inp, dtype):
    """the reference's train-mode query() over every stage, differentiated by autograd -> (values [S,B,Res,N], grads dict)"""
    net = ns.PIFuNetC() if c["chans"] == spec.C_CHANNELS else ns.PIFuNetG()
    if c["chans"] not in (spec.G_CHANNELS, spec.C_CHANNELS):
        net.surface_classifier = ns.SurfaceClassifier(c["chans"], 1, False, nn.Sigmoid())
    if inp["proj"] == "perspective":
        net.projection = ns.perspective
    net.surface_classifier.load_state_dict(
        {**{"filters.%d.weight" % l: W[:, :, None].clone() for l, W in enumerate(inp["Ws"])},
         **{"filters.%d.bias" % l: b.clone() for l, b in enumerate(inp["bs"])}})
    net = net.to(dtype).train()
    fs = [f.to(dtype).clone().requires_grad_() for f in inp["feats"]]
    p = inp["points"].to(dtype).clone().requires_grad_()
    cal = inp["calib"].to(dtype) if inp["calib"] is not None else None
    preds = net.query([[f] for f in fs], p, calibs=cal)
    assert len(preds) == len(fs)
    gout = inp["grad_output"]
    total = sum((pr * (torch.ones_like(pr) if gout is None else gout[s].to(dtype))).sum() for s, pr in enumerate(preds))
    total.backward()
    head = net.surface_classifier
    grads = dict(dfeat=[f.grad for f in fs], dpoints=p.grad, dW=[f.weight.grad[:, :, 0] for f in head.filters],
                 db=[f.bias.grad for f in head.filters])
    return torch.stack([pr.detach() for pr in preds]), grads


def write_npz(path, arrays):
    """np.savez_compressed with a fixed timestamp on every entry"""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(arrays[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            info.external_attr = 0o600 << 16
            z.writestr(info, buf.getvalue())


def gen_vjp(ns):
    for i, c in enumerate(VJP_CASES):
        inp = make_case_inputs(c)
        v32, g32 = reference_vjp(ns, c, inp, torch.float32)
        v64, g64 = reference_vjp(ns, c, inp, torch.float64)
        # the restatement of tests/vjp_cases.py against the reference in fp64
        m64 = query_vjp_ref(inp["feats"], inp["points"], inp["calib"], inp["Ws"], inp["bs"], inp["last_op"], inp["proj"],
                            inp["grad_output"], dtype=torch.float64)
        out = dict(chans=np.array(c["chans"], np.int64), last_op=c["last_op"], calib=c["calib"],
                   value=v32.numpy().astype(np.float32), **{k: c[k] for k in ("B", "S", "N", "H", "W", "gseed", "wseed",
                                                                             "fseed", "pseed")})
        line = []
        for j, g in enumerate(GRAD_NAMES):
            a32, a64 = flat(g32[g]), flat(g64[g])
            scale = a64.abs().max().item()
            dist = (a32 - a64).abs().max().item() / scale
            assert (flat(m64[g]) - a64).abs().max().item() <= 1e-9 * scale, (c["name"], g)
            idx = sample_index(a64.numel(), 1000 * (i + 1) + j)
            out.update({"idx_" + g: idx.numpy().astype(np.int64), g + "64": a64[idx].numpy(),
                        g + "32": a32[idx].numpy().astype(np.float32), "scale_" + g: scale, "dist_" + g: dist})
            line.append("%s %.2e" % (g, dist))
        print("vjp %-24s B=%d S=%d N=%4d %dx%d  |ref32-ref64|/max|g64|: %s" % (
            c["name"], c["B"], c["S"], c["N"], c["H"], c["W"], ", ".join(line)))
        write_npz(os.path.join(HERE, "vjp_%s.npz" % c["name"]), out)


if __name__ == "__main__":
    torch.set_num_threads(8)
    gen_vjp(load_reference())
    print("done")
