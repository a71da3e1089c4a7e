"""The point-gradient goldens (tests/golden/grad_*.npz: the reference's query() differentiated by autograd with respect to the
points), the regeneration of the seeded inputs they do not store, and `query_grad_ref`, a differentiable restatement of
query() built from the oracle's pieces."""
import glob
import os

import numpy as np
import torch

from oracle import spec
from helpers import GOLDEN, checksum
from shape_cases import load_shape_grad_case


def query_grad_ref(feat, points, calib, Ws, bs, last_op, projection="orthogonal", z_scale=spec.Z_SCALE, grad_output=None,
                   dtype=torch.float32):
    """oracle.spec.query_ref without its no_grad, differentiated with respect to the points by autograd, in `dtype`.
    feat [1,C,H,W] or [C,H,W]; points [1,3,N] or [3,N]; calib [1,4,4]/[4,4]/[3,4]/None; grad_output [Res,N] or None (ones)
    -> (value [Res,N], d sum(grad_output * value) / d points [3,N]), both in `dtype`."""
    feat = (feat[0] if feat.dim() == 4 else feat).to(dtype)
    points = (points[0] if points.dim() == 3 else points).to(dtype).detach().clone().requires_grad_(True)
    if calib is not None:
        calib = (calib[0] if calib.dim() == 3 else calib).to(dtype)
    Ws = [w.to(dtype) for w in Ws]
    bs = [b.to(dtype) for b in bs]
    with torch.enable_grad():
        xyz = spec.project_ref(points, calib, projection)
        u, v, z = xyz[0], xyz[1], xyz[2]
        in_img = (u >= -1.0) & (u <= 1.0) & (v >= -1.0) & (v <= 1.0)              # MonoPortNet.py:74
        x = torch.cat([spec.bilinear_ref(feat, u, v), (z * z_scale)[None]], 0)    # :82-83, DepthNormalizer.py:32
        out = in_img.to(dtype)[None] * spec.mlp_ref(x, Ws, bs, last_op)            # :86-89
        g = torch.ones_like(out) if grad_output is None else grad_output.to(dtype)
        (dp,) = torch.autograd.grad(out, points, grad_outputs=g)
    return out.detach(), dp


def grad_cases():
    return sorted(os.path.basename(p)[len("grad_"):-4] for p in glob.glob(os.path.join(GOLDEN, "grad_*.npz")))


def load_grad_case(name):
    """-> dict(points [1,3,N], calib [1,4,4]|None, value [Res,N], grad32 / grad64 [3,N] (the reference's fp32 / fp64 autograd
    gradients), grad_output [Res,N]|None, feat, Ws, bs, last_op, proj, net)"""
    g = np.load(os.path.join(GOLDEN, "grad_%s.npz" % name))
    net = str(g["net"])
    chans = spec.G_CHANNELS if net == "G" else spec.C_CHANNELS
    Ws, bs = spec.make_weights(chans, int(g["wseed"]))
    hw = int(g["hw"])
    feat = spec.make_feat(chans[0] - 1, hw, hw, int(g["fseed"]), float(g["fscale"]))
    # RNG drift must fail loudly, not as a parity error
    np.testing.assert_allclose(np.stack([checksum(w) for w in Ws]), g["w_checksum"], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(checksum(feat), g["f_checksum"], rtol=1e-12, atol=1e-12)
    calib = torch.from_numpy(g["calib"]) if g["calib"].size else None
    gout = torch.from_numpy(g["grad_output"]) if g["grad_output"].size else None
    return dict(name=name, net=net, points=torch.from_numpy(g["points"]), calib=calib, value=torch.from_numpy(g["value"]),
                grad32=torch.from_numpy(g["grad32"]), grad64=torch.from_numpy(g["grad64"]), grad_output=gout, Ws=Ws, bs=bs,
                feat=feat, chans=chans, last_op=spec.LAST_SIGMOID if net == "G" else spec.LAST_TANH, proj=str(g["proj"]))


def within_bar(got, ref):
    """The error bar of the point gradient against the reference's fp32 autograd gradient `ref` ([3,N]): every component
    within 1e-3 * max|ref|, and 99 % of them within 2e-5 * max|ref|.  (The reference's own fp32 gradient differs from its
    fp64 one by up to ~1e-4 * max|g| at leaky-ReLU and texel kinks.)  -> (ok, message)"""
    scale = ref.abs().max().item()
    err = (got.double() - ref.double()).abs()
    frac = (err <= 2e-5 * scale).double().mean().item()
    worst = err.max().item() / scale
    return worst <= 1e-3 and frac >= 0.99, "max|err|/max|g| = %.2e, fraction within 2e-5: %.4f" % (worst, frac)


# ---- the tensor-core gradient program (query_jvp_kernel) -------------------------------------------------------------------
# the first 8 points of every case are border_points(): on the image border / corners and far outside
GOLDEN_CASES = [("grad", "g_rot", 64), ("grad", "g_persp", 48), ("grad", "g_nocalib", 48), ("grad", "g_bigfeat", 48),
                ("grad", "c_rot", 32), ("shape", "g_wide", 72), ("shape", "g_tiny", 72)]


def load_golden(kind, name):
    """a case of GOLDEN_CASES: kind "grad" (tests/golden/grad_*.npz) or "shape" (shape_grad_*.npz)"""
    return load_grad_case(name) if kind == "grad" else load_shape_grad_case(name)


# Goldens on which the fp16 restatement (tc_jvp_ref, all points of the golden) does not pass the bar below with a 2x margin
# get its own distance from grad64 + 10 % as their bar: shape_grad_g_wide's largest component is 2.85e-2 max|g| away
# (a leaky-ReLU kink taken on the other side in fp16).  Every other golden keeps the bar (DESIGN.md, section F1 triple-prime).
MAX_BAR = {"g_wide": 3.1e-2}


def tc_bar(got, g64, name=None):
    """The error bar of the tensor-core gradient against the reference's fp64 gradient: median <= 5e-5 max|g|, 99 % of the
    components <= 5e-3 max|g|, every component <= 5e-2 max|g| (MAX_BAR for the goldens named there).  (The tail comes
    from fp16 taking the other side of a leaky-ReLU kink.)  -> (ok, message)"""
    scale = g64.abs().max().item()
    err = (got.double() - g64.double()).abs().flatten() / scale
    med, p99, worst = err.median().item(), torch.quantile(err, 0.99).item(), err.max().item()
    return (med <= 5e-5 and p99 <= 5e-3 and worst <= MAX_BAR.get(name, 5e-2),
            "|err|/max|g|: median %.2e, p99 %.2e, max %.2e" % (med, p99, worst))
