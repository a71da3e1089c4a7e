"""Quick GPU check of the tensor-core query kernel against the oracle (small sizes first so a hang shows early)."""
import sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from oracle import spec
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
from helpers import build_net

Ws, bs = spec.make_weights(spec.G_CHANNELS, 1234)
feat = spec.make_feat(256, 128, 128, 77)
cal = spec.scene_calib(20, -50)
net = build_net("G", Ws, bs)
print("tc supported:", net.surface_classifier.tc_supported(), flush=True)
net.precision = "tc"
for n in (128, 100, 1000, 20000, 148 * 128 * 3 + 17):
    pts = spec.make_points(n, 5 + n)
    want = spec.query_ref(feat, pts, cal, Ws, bs, spec.LAST_SIGMOID)[0]
    got = net.query([[feat.cuda()]], pts.cuda(), calibs=cal.cuda())[0][0, 0]
    torch.cuda.synchronize()
    err = (got.cpu() - want).abs()
    print("n=%7d  max|tc - oracle| = %.3e  mean = %.3e  zeros-exact=%s" % (n, err.max().item(), err.mean().item(),
          bool(torch.equal(got.cpu()[want == 0], want[want == 0]))), flush=True)
    if err.max().item() > 1e-3:
        bad = err.argmax().item()
        print("  worst idx", bad, got[bad].item(), want[bad].item(), "first 8:", got[:8].tolist(), want[:8].tolist())
# timing: dense 257^3
R = 257
for mode in ("tc",):
    net.precision = mode
    f = feat.cuda(); c = cal.cuda()
    vol = net.query_grid(f, c, R, (-1, -1, -1), (1, 1, 1))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(3):
        vol = net.query_grid(f, c, R, (-1, -1, -1), (1, 1, 1))
    torch.cuda.synchronize()
    dt = (time.perf_counter() - t0) / 3
    print("dense 257^3 [%s]: %.2f ms  -> %.1f Mpts/s, %.1f TFLOP/s algorithmic" % (mode, dt * 1e3, R**3 / dt / 1e6, R**3 * 2363906 / dt / 1e12), flush=True)
