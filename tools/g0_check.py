"""GPU check of the G0 GEMM (layer 0 hoisted to texels) vs. the oracle at several sizes, and the cost
of one per-frame refresh (query after a feature upload vs. query on an unchanged feature map)."""
import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
from oracle import spec
from helpers import build_net

Ws, bs = spec.make_weights(spec.G_CHANNELS, 1234)
feat = spec.make_feat(256, 128, 128, 77)
cal = spec.scene_calib(20, -50)
net = build_net("G", Ws, bs)
net.precision = "tc_v3"
out = {}
for n in (100, 1000, 20000, 148 * 128 * 3 + 17):
    pts = spec.make_points(n, 5 + n)
    want = spec.query_ref(feat, pts, cal, Ws, bs, spec.LAST_SIGMOID)[0]
    got = net.query([[feat.cuda()]], pts.cuda(), calibs=cal.cuda())[0][0, 0]
    torch.cuda.synchronize()
    out[n] = got.cpu()
    err = (got.cpu() - want).abs()
    print("n=%7d  max|v3 - oracle| = %.3e  mean = %.3e" % (n, err.max().item(), err.mean().item()), flush=True)
# cost of a G0 refresh: small query with / without a feature re-upload
f = feat.cuda(); c = cal.cuda()
pts = spec.make_points(4096, 3).cuda()
def run(reupload, iters=50):
    fs = [f.clone() for _ in range(2)]
    for i in range(5):
        net.query([[fs[i % 2] if reupload else f]], pts, calibs=c)
    torch.cuda.synchronize()
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        net.query([[fs[i % 2] if reupload else f]], pts, calibs=c)
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3
a = run(False); b = run(True)
print("4096-point query: %.1f us cached G0, %.1f us with feature upload + G0 refresh (transpose + GEMM)" % (a, b))
