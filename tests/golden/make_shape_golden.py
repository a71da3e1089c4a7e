#!/usr/bin/env python
"""Generate tests/golden/shape_*.npz by running the UNMODIFIED reference (/root/reference) on CPU, on feature maps that are
not square, whose texel count is not a multiple of 128, that sit at or just above the tensor-core program's limit of 65536
texels, or that have an axis of length 1.

Run in the build container (the reference tree does not exist on the GPU box):
    python tests/golden/make_shape_golden.py

Like tests/golden/make_golden.py (whose helpers this uses), the large inputs are not stored but regenerated from seeds; each
file stores checksums of the regenerated tensors.  The files are written with fixed zip timestamps, so a rerun reproduces
them byte for byte.

Three kinds of file:
  shape_<case>.npz       the reference's query() of one map (points, calib, expected; expected64: the same in float64)
  shape_grad_<case>.npz  its point gradient by autograd, in fp32 and fp64 (as tests/golden/make_grad_golden.py)
  shape_batch_<case>.npz its query() over a batch of B maps (as tests/golden/make_batch_golden.py)
The points of every case are, in order: border_points() (8), a cluster whose projections land on and next to the last row
and the last column of the map -- the texels of the last, partial 128-texel block of the per-texel G0 kernel --, then
uniform points.
"""
import io
import os
import sys
import zipfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, os.path.join(HERE, "..", ".."))

from oracle import spec  # noqa: E402
from oracle.ref_loader import load_reference  # noqa: E402
from make_golden import border_points, checksum, load_head, make_calib  # noqa: E402
from make_batch_golden import batch_calib  # noqa: E402
from make_grad_golden import reference_grad  # noqa: E402
from grad_cases import query_grad_ref  # noqa: E402

N_CORNER = 64          # points of the last-texels cluster, after the 8 border points

SHAPE_CASES = [
    # name, net, H, W, wseed, fseed, pseed, N, calib, projection
    dict(name="g_wide", net="G", H=72, W=136, wseed=401, fseed=402, pseed=403, N=2049, calib="rot33", proj="orthogonal"),
    dict(name="g_tall", net="G", H=136, W=72, wseed=401, fseed=412, pseed=413, N=2049, calib="none", proj="orthogonal"),
    dict(name="g_tiny", net="G", H=5, W=7, wseed=421, fseed=422, pseed=423, N=2049, calib="persp", proj="perspective"),
    dict(name="g_row", net="G", H=1, W=200, wseed=431, fseed=432, pseed=433, N=2049, calib="none", proj="orthogonal"),
    dict(name="g_col", net="G", H=200, W=1, wseed=441, fseed=442, pseed=443, N=2049, calib="rot33", proj="orthogonal"),
    dict(name="g_limit", net="G", H=256, W=256, wseed=451, fseed=452, pseed=453, N=2049, calib="rot33", proj="orthogonal"),
    dict(name="g_limit_wide", net="G", H=128, W=512, wseed=461, fseed=462, pseed=463, N=2049, calib="none", proj="orthogonal"),
    dict(name="g_over", net="G", H=257, W=256, wseed=471, fseed=472, pseed=473, N=2049, calib="rot33", proj="orthogonal"),
    dict(name="c_wide", net="C", H=88, W=120, wseed=481, fseed=482, pseed=483, N=2049, calib="rot33", proj="orthogonal"),
    dict(name="c_over", net="C", H=260, W=256, wseed=491, fseed=492, pseed=493, N=2049, calib="rot33", proj="orthogonal"),
]
GRAD_CASES = ["g_wide", "g_tiny"]
BATCH_CASES = [
    # name, net, H, W, wseed, per-image (fseed, pseed), N, calib kind of make_batch_golden.batch_calib, projection
    dict(name="g_wide_persp", net="G", H=72, W=136, wseed=501, images=[(502, 503), (504, 505), (506, 507)], N=2049,
         calib="persp", proj="perspective"),
]


def save_npz(path, **arrays):
    """np.savez_compressed with fixed zip timestamps: the same arrays give the same bytes"""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for k, v in arrays.items():
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(v), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())


def corner_points(H, W, calib, proj, n, seed):
    """n world points [1,3,n] whose projections fall on the last texels of an H x W map in row-major order.  The first half
    lies in the cells just before a texel of the last 128-texel block (so that its far bilinear tap is that texel); the second
    half at pixel coordinates (W-1-a, H-1-b) with a, b in [0, 2), among them the exact corner (u, v) = (1, 1) and the two
    last-texel edges.  An axis of length 1 takes any coordinate in [-1, 1] (all of them land on its one texel).
    Through a calibration, the projection's fp32 rounding differs between implementations: there the points keep 1e-3 pixel
    away from the image border and from texel edges, where a one-ulp difference would flip the mask or the gradient."""
    g = torch.Generator().manual_seed(int(seed))
    f64 = dict(generator=g, dtype=torch.float64)
    eps = 0.0 if calib is None else 1e-3
    h = n // 2
    last = H * W - (H * W - 1) // 128 * 128                      # texels of the last block
    t = H * W - 1 - (torch.rand(h, **f64) * last).floor()
    ix = torch.cat([t % W - torch.rand(h, **f64), W - 1 - torch.rand(n - h, **f64) * 2.0])
    iy = torch.cat([(t / W).floor() - torch.rand(h, **f64), H - 1 - torch.rand(n - h, **f64) * 2.0])
    ix[h:h + 4] = W - 1 - torch.tensor([0.0, 0.0, 1.0, 0.5], dtype=torch.float64) - eps
    iy[h:h + 4] = H - 1 - torch.tensor([0.0, 1.0, 0.0, 0.0], dtype=torch.float64) - eps
    u = 2.0 * ix.clamp(eps, W - 1 - eps) / (W - 1) - 1.0 if W > 1 else torch.rand(n, **f64) * 2 - 1
    v = 2.0 * iy.clamp(eps, H - 1 - eps) / (H - 1) - 1.0 if H > 1 else torch.rand(n, **f64) * 2 - 1
    u, v = u.clamp(-1, 1), v.clamp(-1, 1)
    z = torch.rand(n, **f64) - 0.5
    if calib is None:
        return torch.stack([u, v, z])[None].float()
    m = calib[0].double()
    if proj == "perspective":
        d = 3.0 + z                                   # depth in front of the camera (the persp calib puts z near 3)
        p = torch.stack([u * d, v * d, d])
    else:
        p = torch.stack([u, v, z])
    return torch.linalg.solve(m[:3, :3], p - m[:3, 3:4])[None].float()


def case_points(H, W, calib, proj, N, seed):
    pts = spec.make_points(N, seed).clone()
    pts[:, :, 8:8 + N_CORNER] = corner_points(H, W, calib, proj, N_CORNER, seed + 1000)
    return border_points(pts)


def make_net(ns, net, proj, Ws, bs):
    m = (ns.PIFuNetG() if net == "G" else ns.PIFuNetC()).eval()
    if proj == "perspective":
        m.projection = ns.perspective
    load_head(m, Ws, bs)
    return m


def case_inputs(c):
    chans = spec.G_CHANNELS if c["net"] == "G" else spec.C_CHANNELS
    last_op = spec.LAST_SIGMOID if c["net"] == "G" else spec.LAST_TANH
    Ws, bs = spec.make_weights(chans, c["wseed"])
    return chans, last_op, Ws, bs


@torch.no_grad()
def gen_shape_query(ns):
    for c in SHAPE_CASES:
        chans, last_op, Ws, bs = case_inputs(c)
        feat = spec.make_feat(chans[0] - 1, c["H"], c["W"], c["fseed"])
        calib = make_calib(c["calib"])
        pts = case_points(c["H"], c["W"], calib, c["proj"], c["N"], c["pseed"])
        net = make_net(ns, c["net"], c["proj"], Ws, bs)
        decoy = torch.zeros_like(feat)
        out = net.query([[decoy], [decoy], [decoy], [feat]], pts, calibs=calib)
        assert len(out) == 1
        ref = out[0][0].numpy()
        mine = spec.query_ref(feat, pts, calib, Ws, bs, last_op, c["proj"]).numpy()
        err = np.abs(ref - mine).max()
        corner_in = (ref[0, 8:8 + N_CORNER] != 0).mean()
        print("shape %-12s %3d x %3d  N=%5d  in-img %.2f (corner cluster %.2f)  |oracle-ref| = %.2e" % (
            c["name"], c["H"], c["W"], c["N"], (ref[0] != 0).mean(), corner_in, err))
        assert err < 2e-6
        assert corner_in > 0.9, "the corner cluster must land in the image"
        # the reference in float64 (head, map, points and calib converted): how far its own fp32 result is from exact
        net64 = make_net(ns, c["net"], c["proj"], Ws, bs).double()
        f64 = feat.double()
        ref64 = net64.query([[f64]], pts.double(), calibs=calib.double() if calib is not None else None)[0][0].numpy()
        print("      %-12s |ref32 - ref64| = %.2e" % (c["name"], np.abs(ref - ref64).max()))
        save_npz(os.path.join(HERE, "shape_%s.npz" % c["name"]),
                 kind="query", points=pts.numpy(), calib=(calib.numpy() if calib is not None else np.zeros((0,), np.float32)),
                 expected=ref, expected64=ref64, net=c["net"], wseed=c["wseed"], fseed=c["fseed"], H=c["H"], W=c["W"],
                 proj=c["proj"],
                 w_checksum=np.stack([checksum(w) for w in Ws]), f_checksum=checksum(feat))


def gen_shape_grad(ns):
    for c in (c for c in SHAPE_CASES if c["name"] in GRAD_CASES):
        chans, last_op, Ws, bs = case_inputs(c)
        feat = spec.make_feat(chans[0] - 1, c["H"], c["W"], c["fseed"])
        calib = make_calib(c["calib"])
        pts = case_points(c["H"], c["W"], calib, c["proj"], c["N"], c["pseed"])
        val32, g32 = reference_grad(ns, c, Ws, bs, feat, pts, calib, None, torch.float32)
        _, g64 = reference_grad(ns, c, Ws, bs, feat, pts, calib, None, torch.float64)
        mv, m32 = query_grad_ref(feat, pts, calib, Ws, bs, last_op, c["proj"])
        _, m64 = query_grad_ref(feat, pts, calib, Ws, bs, last_op, c["proj"], dtype=torch.float64)
        scale = g64.abs().max().item()
        print("shape grad %-8s %3d x %3d  max|g| %.3g  |ref32-ref64|/max %.2e  |oracle64-ref64|/max %.2e  "
              "|oracle32-ref32|/max %.2e  |oracle value - ref| %.2e" % (
                  c["name"], c["H"], c["W"], scale, (g32.double() - g64).abs().max().item() / scale,
                  (m64 - g64).abs().max().item() / scale, (m32 - g32).abs().max().item() / scale,
                  (mv - val32).abs().max().item()))
        assert (mv - val32).abs().max().item() < 2e-6
        assert (m64 - g64).abs().max().item() <= 1e-9 * scale
        save_npz(os.path.join(HERE, "shape_grad_%s.npz" % c["name"]),
                 kind="grad", points=pts.numpy(), calib=(calib.numpy() if calib is not None else np.zeros((0,), np.float32)),
                 value=val32.numpy(), grad32=g32.numpy(), grad64=g64.numpy(), net=c["net"], wseed=c["wseed"],
                 fseed=c["fseed"], H=c["H"], W=c["W"], proj=c["proj"], w_checksum=np.stack([checksum(w) for w in Ws]),
                 f_checksum=checksum(feat))


@torch.no_grad()
def gen_shape_batch(ns):
    for c in BATCH_CASES:
        chans, last_op, Ws, bs = case_inputs(c)
        feats = [spec.make_feat(chans[0] - 1, c["H"], c["W"], fs) for fs, _ in c["images"]]
        cals = [batch_calib(c["calib"], b) for b in range(len(c["images"]))]
        pts = [case_points(c["H"], c["W"], cals[b], c["proj"], c["N"], ps) for b, (_, ps) in enumerate(c["images"])]
        feat, points = torch.cat(feats, 0), torch.cat(pts, 0)
        calib = torch.cat(cals, 0) if cals[0] is not None else None
        net = make_net(ns, c["net"], c["proj"], Ws, bs)
        decoy = torch.zeros_like(feat)
        out = net.query([[decoy], [decoy], [decoy], [feat]], points, calibs=calib)
        assert len(out) == 1
        ref = out[0].numpy()
        err = max(np.abs(ref[b] - spec.query_ref(feats[b], pts[b], cals[b], Ws, bs, last_op, c["proj"]).numpy()).max()
                  for b in range(len(feats)))
        print("shape batch %-12s B=%d %3d x %3d  N=%5d  |oracle per image - ref| = %.2e" % (
            c["name"], len(feats), c["H"], c["W"], c["N"], err))
        assert err < 2e-6
        save_npz(os.path.join(HERE, "shape_batch_%s.npz" % c["name"]),
                 kind="batch", points=points.numpy(), calib=(calib.numpy() if calib is not None else np.zeros((0,), np.float32)),
                 expected=ref, net=c["net"], wseed=c["wseed"], fseeds=np.array([i[0] for i in c["images"]]), H=c["H"],
                 W=c["W"], proj=c["proj"], w_checksum=np.stack([checksum(w) for w in Ws]),
                 f_checksum=np.stack([checksum(f) for f in feats]))


if __name__ == "__main__":
    torch.set_num_threads(8)
    ns = load_reference()
    gen_shape_query(ns)
    gen_shape_grad(ns)
    gen_shape_batch(ns)
    print("done")
