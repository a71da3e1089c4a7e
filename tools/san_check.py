"""Tiny invocation of every kernel family for compute-sanitizer (memcheck): both tensor-core programs, the fp32 kernel and
its point-gradient kernel (single maps and batches), the octree engine (eager, and a captured lossless frame), marching
cubes, the visible-surface kernel and the enqueue-only renders of captured frames (mp_colorize_surface_async on both
programs, mp_render_normals_async)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np, torch
from oracle import spec
from helpers import build_net
from monoport_b200.engine import Seg3dLossless, Seg3dTopk, make_query_func
from monoport_b200.recon import forward_vertices, marching_cubes
Ws, bs = spec.make_weights(spec.G_CHANNELS, 3)
feat = spec.make_feat(256, 128, 128, 4, 0.5)
Ws, bs, feat, _ = spec.heightfield_person(Ws, bs, feat)
net = build_net("G", Ws, bs)
cal = spec.scene_calib(20, 33).cuda()
pts = spec.make_points(700, 1).cuda()
for mode in ("fp32", "tc"):
    net.precision = mode
    out = net.query([[feat.cuda()]], pts, calibs=cal)[0]
    torch.cuda.synchronize()
    print(mode, float(out.sum()))
net.precision = "tc"
b = np.array([[-1.0, -1.0, -1.0]], dtype=np.float32)
for faster in (True, False):
    eng = Seg3dLossless(make_query_func(net), b, -b, [9, 17, 33], balance_value=0.5, faster=faster).to("cuda")
    sdf = eng(im_feat_list=[[feat.cuda()]], calib_tensor=cal)
    print("engine faster=%s" % faster, eng.last_stats, None if sdf is None else float(sdf.sum()))
# a captured lossless frame: the conflict loop of every level as a WHILE node decided on the device
from monoport_b200.pipeline import FrameGraph
eng = Seg3dLossless(make_query_func(net), b, -b, [9, 17, 33], balance_value=0.5, faster=False).to("cuda")
fg = FrameGraph(net, eng, cal.cpu(), "front", with_encoder=False)
sdf = fg.launch(feat.cuda()).result()[0]
print("captured lossless frame", fg.last_stats, fg.last_conflict_loops, None if sdf is None else float(sdf.sum()))
fg.close()
eng = Seg3dTopk(make_query_func(net), b, -b, [9, 17, 33], num_points=[0, 500, 2000]).to("cuda")
sdf = eng(im_feat_list=[[feat.cuda()]], calib_tensor=cal)
X, Y, Z, n = forward_vertices(sdf, "front")
v, f = marching_cubes(sdf[0, 0])
torch.cuda.synchronize()
# the colour head's tensor-core program incl. the fused direct rendering, and a frame outside the range guard's limit
from monoport_b200.recon import colorization
cW, cb = spec.make_weights(spec.C_CHANNELS, 5)
netC = build_net("C", cW, cb)
featC = spec.make_feat(512, 128, 128, 6, 0.5).cuda()
img = colorization(netC, [[featC]], X, Y, Z, cal, resolution=33)
# the enqueue-only renders of captured frames: counts on the device (capacity R*R, the tail past the count unread), the
# colour render in range (tensor cores) and out of range (the exact twin)
import ctypes
from monoport_b200 import _lib
lib = _lib.load()
k = X.numel()
Xb, Yb = torch.zeros(33 * 33, dtype=torch.int64, device="cuda"), torch.zeros(33 * 33, dtype=torch.int64, device="cuda")
Zb, Nb = torch.zeros(33 * 33, device="cuda"), torch.zeros(33 * 33, 3, device="cuda")
Xb[:k], Yb[:k], Zb[:k], Nb[:k] = X, Y, Z, n
cnt = torch.tensor([k], dtype=torch.int64, device="cuda")
canv = torch.ones(33, 33, 3, device="cuda")
P = lambda t: ctypes.c_void_p(t.data_ptr())
_lib.check(lib.mp_render_normals_async(P(Xb), P(Yb), P(Nb), P(cnt), 33 * 33, 33, P(canv), _lib.stream_ptr()), "normals")
for fc in (featC, featC * 60.0):
    fh = netC.feature_handle(fc)
    _lib.check(lib.mp_colorize_surface_async(netC.surface_classifier.handle(), fh.ptr, P(Xb), P(Yb), P(Zb), P(cnt), 33 * 33, 33,
                                             _lib.f3([-1, -1, -1]), _lib.f3([1, 1, 1]), _lib.calib12(cal), 0,
                                             ctypes.c_float(netC.normalizer.scale), _lib.MODE_AUTO, P(canv), _lib.stream_ptr()),
               "colour async")
    torch.cuda.synchronize()
print("async renders", float(canv.sum()))
big = net.query([[feat.cuda() * 60.0]], pts, calibs=cal)[0]
# batched queries (one launch over B images) in every mode; image 1 is outside the range guard's limit, so the guarded
# modes split the launch per image between the tensor-core and the exact kernel
fb = torch.cat([feat, feat * 60.0, spec.make_feat(256, 128, 128, 8, 0.5)], 0).cuda()
pb = torch.cat([spec.make_points(100, 2), spec.make_points(100, 3), spec.make_points(100, 4)], 0).cuda()
cb = torch.cat([spec.scene_calib(20, 33), spec.scene_calib(-10, 5), spec.scene_calib(30, 70)], 0).cuda()
for mode in ("fp32", "tc", "auto"):
    net.precision = mode
    ob = net.query([[fb]], pb, calibs=cb)[0]
    torch.cuda.synchronize()
    print("batch", mode, float(ob.sum()))
# the batched point gradient (one launch of each program over the three images): in "tc" image 1 is differentiated by the
# exact kernel, the others by the tensor-core program
for precision in ("fp32", "tc"):
    vb, db = net.query_gradient([[fb]], pb, calibs=cb, precision=precision)
    torch.cuda.synchronize()
    print("batch grad", precision, float(db.abs().sum()))
# the point-gradient kernel: geometry head (ragged last tile), colour head with a grad_output and [N,3]-strided points
vg, dg = net.query_gradient([[feat.cuda()]], pts[:, :, :123], calibs=cal)
pv = pts[0, :, :77].t().contiguous().t()[None]
vc, dc = netC.query_gradient([[featC]], pv, calibs=cal, grad_output=torch.randn(1, 3, 77, device="cuda"))
torch.cuda.synchronize()
print("grad", float(dg.abs().sum()), float(dc.abs().sum()))
torch.cuda.synchronize()
print("ok", X.numel(), v.shape, f.shape, float(img.sum()), float(big.sum()))
