"""MonoPortNet with the reference's API (monoport/lib/modeling/MonoPortNet.py) whose eval-mode `query()` is ONE
fused sm_90a kernel launch (project -> mask -> bilinear gather -> z-concat -> 5-layer skip MLP -> last_op -> mask)
through the C-ABI of libmonoport_b200.  There is no PyTorch / CPU fallback for query(): CPU tensors or a missing
library raise."""
import ctypes
import os
import threading

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.autograd.function import once_differentiable

from .. import _lib
from ..config import CN
from .geometry import index, orthogonal, perspective  # noqa: F401  (re-exported like the reference)
from .normalizers import DepthNormalizer, PIFuNomalizer  # noqa: F401
from .backbones import HGFilter, PIFuHGFilters, ResnetFilter, PIFuResBlkFilters  # noqa: F401
from .heads import SurfaceClassifier, PIFuNetGMLP, PIFuNetCMLP  # noqa: F401

_MODES = {"fp32": _lib.MODE_FP32, "tc": _lib.MODE_TC, "auto": _lib.MODE_AUTO, "tc_v3": _lib.MODE_TC_V3}


class FeatureHandle:
    """Device-side channel-last copy of one [1,C,H,W] feature map, or of the B maps of a [B,C,H,W] batch (mp_feat_t)."""

    def __init__(self, C, H, W, device, B=1):
        self.shape = (C, H, W)
        self.batch = B
        self.device = device
        self.ptr = ctypes.c_void_p()
        with _lib.device_guard(device):
            if B == 1:
                _lib.check(_lib.load().mp_feat_create(C, H, W, ctypes.byref(self.ptr)), "mp_feat_create")
            else:
                _lib.check(_lib.load().mp_feat_create_batch(B, C, H, W, ctypes.byref(self.ptr)), "mp_feat_create_batch")
        self.key = None
        self._src = None
        self._scope = 0

    def upload(self, feat, trust_identity=False):
        """Repack `feat` into the handle.  The upload is skipped only when (storage address, version counter) are
        unchanged AND that identity may be trusted: inside one `_lib.frame_scope()` (the levels of one engine call) or
        when the application opted in (`MonoPortNet.feature_cache = True`).  Writes that bypass the version counter
        (CUDA-graph static buffers, custom kernels, NCCL receives) are otherwise re-uploaded: ~11 us repack + ~26 us G0."""
        key = _lib.tensor_identity(feat)          # None for inference-mode tensors: never matches
        sid = _lib.current_scope()
        if key is not None and key == self.key and (trust_identity or _lib.TRUST_TENSOR_IDENTITY or (sid != 0 and sid == self._scope)):
            return
        f = feat.detach()
        if (f.dtype == torch.float32 and f.shape[1] > 1 and not f.is_contiguous()
                and f.is_contiguous(memory_format=torch.channels_last)):
            # a channels_last encoder already emits [H,W,C]: the kernels read it in place -- no repack, no copy (SURVEY.md
            # §8f-3).  `_src` below keeps the tensor alive for the frame.
            _lib.check(_lib.load().mp_feat_bind_nhwc(self.ptr, ctypes.c_void_p(f.data_ptr()), _lib.stream_ptr(self.device)),
                       "mp_feat_bind_nhwc")
        else:
            if f.dtype != torch.float32 or not f.is_contiguous():
                f = f.to(torch.float32).contiguous()
            _lib.check(_lib.load().mp_feat_upload(self.ptr, ctypes.c_void_p(f.data_ptr()), 1, _lib.stream_ptr(self.device)),
                       "mp_feat_upload")
        # `_src` keeps the tensor alive so the caching allocator cannot hand its address to the NEXT frame's features
        self.key, self._src, self._scope = key, feat, sid

    def invalidate(self):
        self.key = None
        self._src = None

    def __del__(self):
        try:
            if self.ptr:
                _lib.load().mp_feat_destroy(self.ptr)
        except Exception:
            pass


class _QueryStage(torch.autograd.Function):
    """One stage of MonoPortNet.query_stages: the exact fp32 query in the forward, mp_query_points_vjp in the backward --
    d features, d points and the head's d weights / d biases, each only when autograd asks for it."""

    @staticmethod
    def forward(ctx, net, feat, points, calibs, *params):
        ctx.net = net
        ctx.has_calibs = calibs is not None
        ctx.save_for_backward(feat, points, *([calibs] if calibs is not None else []), *params)
        return net._query_fp32(feat, points, calibs)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad):
        saved = ctx.saved_tensors            # (raises if an optimizer step changed the head since the forward)
        feat, points = saved[0], saved[1]
        calibs = saved[2] if ctx.has_calibs else None
        want_feat, want_points = ctx.needs_input_grad[1], ctx.needs_input_grad[2]
        want_head = any(ctx.needs_input_grad[4:])
        dfeat, dpoints, dws, dbs = ctx.net._query_vjp(feat, points, calibs, grad, want_feat, want_points, want_head,
                                                      torch.are_deterministic_algorithms_enabled())
        dparams = [None] * (len(saved) - (3 if ctx.has_calibs else 2))
        if want_head:
            head = ctx.net.surface_classifier
            for l, f in enumerate(head.filters):
                dparams[2 * l] = dws[l].reshape(f.weight.shape).to(f.weight.dtype)
                dparams[2 * l + 1] = dbs[l].to(f.bias.dtype)
        return (None, None if dfeat is None else dfeat.to(feat.dtype),
                None if dpoints is None else dpoints.to(points.dtype), None, *dparams)


class MonoPortNet(nn.Module):
    def __init__(self, opt_net):
        super().__init__()
        self.opt = opt_net
        assert opt_net.projection in ['orthogonal', 'perspective']
        # component choice by name, like the reference (MonoPortNet.py:23-28)
        self.image_filter = globals()[opt_net.backbone.IMF](opt_net.backbone)
        self.surface_classifier = globals()[opt_net.head.IMF](opt_net.head)
        self.projection = globals()[opt_net.projection]
        self.normalizer = globals()[opt_net.normalizer.IMF](opt_net.normalizer)
        # arithmetic of the fused kernel: "auto" (tensor cores when supported), "tc" (= "tc_v3"), "fp32"
        self.precision = os.environ.get("MONOPORT_B200_MODE", "auto")
        # True: skip the per-call feature upload when the tensor's (address, version) are unchanged (see FeatureHandle.upload
        # for what that identity cannot see); default off -- every query()/query_grid()/engine call uploads its frame
        self.feature_cache = os.environ.get("MONOPORT_B200_FEATURE_CACHE", "0") == "1"
        self._feat_handles = {}

    def __getstate__(self):          # feature handles are native, per-thread scratch: a copy starts without them
        d = dict(self.__dict__)
        d["_feat_handles"] = {}
        return d

    # ---- encoder: stays PyTorch ---------------------------------------------------------------------------
    def filter(self, images, feat_prior=None):
        feats_stages = self.image_filter(images)
        if feat_prior is not None:   # netC: prepend netG's last-stage features (MonoPortNet.py:41-45)
            feat_prior = F.interpolate(feat_prior, size=(128, 128))
            feats_stages = [[torch.cat([feat_prior, f], dim=1) for f in feats] for feats in feats_stages]
        return feats_stages

    # ---- the hot path -------------------------------------------------------------------------------------
    def feature_handle(self, feat):
        if feat.dim() != 4 or feat.shape[0] != 1:
            raise ValueError("feature map must be [1,C,H,W] (batch 1, RTL/main.py:175); got %s" % (tuple(feat.shape),))
        if feat.device.type != "cuda":
            raise RuntimeError("monoport_b200.query: features must be CUDA tensors (there is no CPU path)")
        _, C, H, W = feat.shape
        # one handle per calling thread: the handle carries the channel-last copies of the CURRENT frame, and the
        # demo-style pipelines query different frames from different threads (RTL/dataloader.py:734-751)
        key = (C, H, W, feat.device.index, threading.get_ident())
        h = self._feat_handles.get(key)
        if h is None:
            h = self._feat_handles[key] = FeatureHandle(C, H, W, feat.device)
        h.upload(feat, trust_identity=self.feature_cache)
        return h

    def batch_feature_handle(self, feat):
        """The handle of a [B,C,H,W] batch (B > 1) for query(): B maps, evaluated together by mp_query_points_batch.  The
        single-map entry points (feature_handle, the grid queries, the engines) do not take it."""
        B, C, H, W = feat.shape
        key = ("batch", B, C, H, W, feat.device.index, threading.get_ident())
        h = self._feat_handles.get(key)
        if h is None:
            h = self._feat_handles[key] = FeatureHandle(C, H, W, feat.device, B=B)
        h.upload(feat, trust_identity=self.feature_cache)
        return h

    def invalidate_features(self):
        """Forget every uploaded frame (call after writing into a feature tensor behind PyTorch's back)."""
        for h in self._feat_handles.values():
            h.invalidate()

    def _mode(self):
        try:
            return _MODES[self.precision]
        except KeyError:
            raise ValueError("precision must be one of %s" % sorted(_MODES))

    @torch.no_grad()
    def query(self, feats_stages, points, calibs=None, transforms=None):
        """list(list([B,C,H,W])), points [B,3,N], calibs [B,4,4]|[B,3,4]|None -> [ [B,Res,N] ]
        (MonoPortNet.py:48-91, eval mode: only the LAST stage is evaluated, :63-64).  B == 1 is the single-frame path of the
        demo; B > 1 evaluates all images in one launch (mp_query_points_batch)."""
        if self.training:
            raise NotImplementedError("training-mode (multi-stage, autograd) query is outside the accelerated hot path; "
                                      "call .eval() (RTL/main.py:116), or query_stages() for the differentiable query")
        if transforms is not None:
            raise NotImplementedError("`transforms` is not supported (never passed on the recon path, RTL/main.py:179-182)")
        feats = feats_stages[-1]
        if len(feats) != 1:
            raise NotImplementedError("multi-level feature lists (HRNet) are not supported")
        feat = feats[0]
        if feat.device.type != "cuda":
            raise RuntimeError("monoport_b200.query: features must be CUDA tensors (there is no CPU path)")
        if feat.dim() == 4 and feat.shape[0] > 1:
            return self._query_batch(feat, points, calibs)
        if points.dim() != 3 or points.shape[0] != 1 or points.shape[1] != 3:
            raise ValueError("points must be [1,3,N]; got %s" % (tuple(points.shape),))
        if points.device != feat.device:
            raise ValueError("points and features live on different devices")
        if points.dtype != torch.float32:
            points = points.float()
        n = points.shape[2]
        s = points.stride()
        if n > 0 and (s[1] < 1 or s[2] < 1):
            points = points.contiguous()
            s = points.stride()
        head = self.surface_classifier
        res = head.filter_channels[-1]
        out = torch.empty((1, res, n), dtype=torch.float32, device=feat.device)
        if n == 0:
            return [out]
        with _lib.device_guard(feat.device):
            fh = self.feature_handle(feat)
            proj = _lib.PROJ_PERSPECTIVE if self.projection is perspective else _lib.PROJ_ORTHOGONAL
            _lib.check(_lib.load().mp_query_points(
                head.handle(), fh.ptr, ctypes.c_void_p(points.data_ptr()), n, s[1], s[2], _lib.calib12(calibs), proj,
                ctypes.c_float(self.normalizer.scale), ctypes.c_void_p(out.data_ptr()), n, self._mode(),
                _lib.stream_ptr(feat.device)), "mp_query_points")
        return [out]

    @torch.no_grad()
    def query_gradient(self, feats_stages, points, calibs=None, grad_output=None, precision="fp32"):
        """query() and its gradient with respect to the points (mp_query_points_grad_mode).  feats/points/calibs as for
        query() with B == 1; grad_output [1,Res,N] or None (ones).
        precision "fp32" (default): one launch of the exact fp32 kernel; preds bit-identical to query() with precision "fp32".
        "tc": the tensor-core program's forward-mode derivative; preds bit-identical to query() with precision "tc", and a
        frame above the head's feature limit is differentiated exactly (decided on the GPU).  Maps above 65536 texels are
        refused.  "auto": "tc" where the head and the map allow it, else "fp32".
        -> (preds [1,Res,N], dpoints [1,3,N] = d sum(grad_output * preds) / d points; for the geometry head and
            grad_output=None, grad sigma).
        Points outside the image get 0 for both.  Autograd is not involved: `points.requires_grad` is ignored."""
        if precision not in ("fp32", "tc", "auto"):
            raise ValueError("precision must be one of 'fp32', 'tc', 'auto'; got %r" % (precision,))
        if self.training:
            raise NotImplementedError("query_gradient is eval-mode only (the gradient of the last stage, like query()); "
                                      "call .eval()")
        feats = feats_stages[-1]
        if len(feats) != 1:
            raise NotImplementedError("multi-level feature lists (HRNet) are not supported")
        feat = feats[0]
        if feat.device.type != "cuda":
            raise RuntimeError("monoport_b200.query_gradient: features must be CUDA tensors (there is no CPU path)")
        if feat.dim() != 4 or feat.shape[0] != 1:
            raise ValueError("query_gradient takes one feature map [1,C,H,W]; got %s" % (tuple(feat.shape),))
        if points.dim() != 3 or points.shape[0] != 1 or points.shape[1] != 3:
            raise ValueError("points must be [1,3,N]; got %s" % (tuple(points.shape),))
        if points.device != feat.device:
            raise ValueError("points and features live on different devices")
        points = points.detach()
        if points.dtype != torch.float32:
            points = points.float()
        n = points.shape[2]
        s = points.stride()
        if n > 0 and (s[1] < 1 or s[2] < 1):
            points = points.contiguous()
            s = points.stride()
        head = self.surface_classifier
        res = head.filter_channels[-1]
        gout = None
        if grad_output is not None:
            if tuple(grad_output.shape) != (1, res, n):
                raise ValueError("grad_output must be [1,%d,%d]; got %s" % (res, n, tuple(grad_output.shape)))
            if grad_output.device != feat.device:
                raise ValueError("grad_output and features live on different devices")
            gout = grad_output.detach()[0].to(torch.float32).contiguous()
        out = torch.empty((1, res, n), dtype=torch.float32, device=feat.device)
        dp = torch.empty((1, 3, n), dtype=torch.float32, device=feat.device)
        if n == 0:
            return out, dp
        with _lib.device_guard(feat.device):
            fh = self.feature_handle(feat)
            proj = _lib.PROJ_PERSPECTIVE if self.projection is perspective else _lib.PROJ_ORTHOGONAL
            _lib.check(_lib.load().mp_query_points_grad_mode(
                head.handle(), fh.ptr, ctypes.c_void_p(points.data_ptr()), n, s[1], s[2], _lib.calib12(calibs), proj,
                ctypes.c_float(self.normalizer.scale), None if gout is None else ctypes.c_void_p(gout.data_ptr()), n,
                ctypes.c_void_p(out.data_ptr()), n, ctypes.c_void_p(dp.data_ptr()), n, None, _MODES[precision],
                _lib.stream_ptr(feat.device)), "mp_query_points_grad_mode")
        return out, dp

    # ---- training: the differentiable query ---------------------------------------------------------------
    # points per chunk of the weight-gradient contraction (its scratch: about 16 KB per point for the geometry head) and, in
    # torch's deterministic mode, of the ordered feature gradient; the gradients that are bit-reproducible are so for one
    # chunk size
    vjp_chunk_points = 8192

    def query_stages(self, feats_stages, points, calibs=None, transforms=None):
        """list(list([B,C,H,W])), points [B,3,N], calibs [B,4,4]|[B,3,4]|None -> [ [B,Res,N] for every stage ]
        What the reference's train-mode query() computes (MonoPortNet.py:63-91: every hourglass stage), in either module
        mode, differentiable with respect to every stage's feature map, the points and the head's `filters.{l}.weight` /
        `filters.{l}.bias`.  The values are the exact fp32 kernel's (query() with precision "fp32", bit for bit); the
        backward is one fused sm_90a VJP launch per chunk of points plus the weight-gradient contraction
        (mp_query_points_vjp_ex).  The weight, bias and point gradients are bit-reproducible for one `vjp_chunk_points`.
        The feature gradient is accumulated with atomics (like grid_sample's backward) and so is not -- unless torch's
        deterministic mode is on (torch.use_deterministic_algorithms(True), read when the backward runs): then it is summed in
        a fixed order (per chunk of `vjp_chunk_points` points, sorted by cell; DESIGN §F1⁗), the same bits from run to run
        and whichever other gradients are requested, and the other gradients are the same bits as without it.  That covers
        the query's share of a training step only: torch flags some ops of the shipped encoders' backward passes (HG's
        bicubic upsampling, ResBlk's reflection padding) as nondeterministic.  No double backward, no calib gradient."""
        if transforms is not None:
            raise NotImplementedError("`transforms` is not supported (never passed on the recon path, RTL/main.py:179-182)")
        if calibs is not None and calibs.requires_grad:
            raise ValueError("query_stages gives no gradient with respect to calibs; pass calibs.detach()")
        head = self.surface_classifier
        params = [t for f in head.filters for t in (f.weight, f.bias)]
        preds = []
        for feats in feats_stages:
            if len(feats) != 1:
                raise NotImplementedError("multi-level feature lists (HRNet) are not supported")
            feat = feats[0]
            if feat.device.type != "cuda":
                raise RuntimeError("monoport_b200.query_stages: features must be CUDA tensors (there is no CPU path)")
            B = feat.shape[0] if feat.dim() == 4 else -1
            if feat.dim() != 4 or points.dim() != 3 or points.shape[0] != B or points.shape[1] != 3:
                raise ValueError("features must be [B,C,H,W] and points [B,3,N]; got %s and %s"
                                 % (tuple(feat.shape), tuple(points.shape)))
            if calibs is not None and (calibs.dim() != 3 or calibs.shape[0] != B or calibs.shape[1] not in (3, 4)
                                       or calibs.shape[2] != 4):
                raise ValueError("calibs must be [B,4,4] or [B,3,4] with the features' B=%d; got %s"
                                 % (B, tuple(calibs.shape)))
            if points.device != feat.device:
                raise ValueError("points and features live on different devices")
            preds.append(_QueryStage.apply(self, feat, points, calibs, *params))
        return preds

    def _points_rows(self, points):
        p = points.detach()
        if p.dtype != torch.float32:
            p = p.float()
        if p.shape[2] > 0 and min(p.stride()) < 1:
            p = p.contiguous()
        return p

    def _query_fp32(self, feat, points, calibs):
        """the values of query_stages: query() with precision "fp32" (B = 1: mp_query_points, else mp_query_points_batch)"""
        B, n = feat.shape[0], points.shape[2]
        res = self.surface_classifier.filter_channels[-1]
        out = torch.empty((B, res, n), dtype=torch.float32, device=feat.device)
        if n == 0:
            return out
        p = self._points_rows(points)
        s = p.stride()
        proj = _lib.PROJ_PERSPECTIVE if self.projection is perspective else _lib.PROJ_ORTHOGONAL
        with _lib.device_guard(feat.device):
            lib = _lib.load()
            if B == 1:
                fh = self.feature_handle(feat.detach())
                _lib.check(lib.mp_query_points(
                    self.surface_classifier.handle(), fh.ptr, ctypes.c_void_p(p.data_ptr()), n, s[1], s[2],
                    _lib.calib12(None if calibs is None else calibs.detach()), proj, ctypes.c_float(self.normalizer.scale),
                    ctypes.c_void_p(out.data_ptr()), n, _lib.MODE_FP32, _lib.stream_ptr(feat.device)), "mp_query_points")
            else:
                cal = None if calibs is None else calibs.detach()[:, :3, :4].to(device=feat.device, dtype=torch.float32).contiguous()
                fh = self.batch_feature_handle(feat.detach())
                _lib.check(lib.mp_query_points_batch(
                    self.surface_classifier.handle(), fh.ptr, B, ctypes.c_void_p(p.data_ptr()), n, s[0], s[1], s[2],
                    None if cal is None else ctypes.c_void_p(cal.data_ptr()), proj, ctypes.c_float(self.normalizer.scale),
                    ctypes.c_void_p(out.data_ptr()), res * n, n, _lib.MODE_FP32, _lib.stream_ptr(feat.device)),
                    "mp_query_points_batch")
        return out

    def _query_vjp(self, feat, points, calibs, grad, want_feat, want_points, want_head, deterministic=False):
        """-> (d feat [B,C,H,W] | None, d points [B,3,N] | None, [d W_l [Cout,Cin]] | None, [d b_l] | None) of
        sum(grad * query) (mp_query_points_vjp_ex).  deterministic: the feature gradient in a fixed order
        (MP_VJP_DETERMINISTIC), chunked by `vjp_chunk_points` whatever else is requested; the other gradients are the same
        bits either way.  The map is uploaded again: a query since the forward may have replaced the handle's contents."""
        B, C, H, W = feat.shape
        n = points.shape[2]
        head = self.surface_classifier
        dev = feat.device
        f32 = dict(dtype=torch.float32, device=dev)
        dfeat = torch.empty((B, C, H, W), **f32) if want_feat else None
        dpoints = torch.empty((B, 3, n), **f32) if want_points else None
        dws = [torch.empty(f.weight.shape[:2], **f32) for f in head.filters] if want_head else None
        dbs = [torch.empty(f.bias.shape, **f32) for f in head.filters] if want_head else None
        if n == 0:
            for t in [dfeat, dpoints] + (dws or []) + (dbs or []):
                if t is not None:
                    t.zero_()
            return dfeat, dpoints, dws, dbs
        p = self._points_rows(points)
        s = p.stride()
        gout = grad.detach().to(torch.float32).contiguous()
        proj = _lib.PROJ_PERSPECTIVE if self.projection is perspective else _lib.PROJ_ORTHOGONAL
        with _lib.device_guard(dev):
            lib = _lib.load()
            cal = None if calibs is None else calibs.detach()[:, :3, :4].to(**f32).contiguous()
            key = ((C, H, W, dev.index, threading.get_ident()) if B == 1 else
                   ("batch", B, C, H, W, dev.index, threading.get_ident()))
            fh = self._feat_handles.get(key)
            if fh is None:
                fh = self._feat_handles[key] = FeatureHandle(C, H, W, dev, B=B)
            fh.invalidate()
            fh.upload(feat.detach())
            mlp = head.handle()
            flags = _lib.VJP_DETERMINISTIC if deterministic else 0
            nbytes = lib.mp_query_points_vjp_scratch_bytes_ex(mlp, fh.ptr, B, n, int(self.vjp_chunk_points), int(want_feat),
                                                              int(want_head), flags)
            if nbytes < 0:
                _lib.check(int(nbytes), "mp_query_points_vjp_scratch_bytes_ex")
            scratch = torch.empty(int(nbytes), dtype=torch.uint8, device=dev) if nbytes > 0 else None
            L = len(head.filters)
            ptrs = (lambda ts: None if ts is None else (ctypes.c_void_p * L)(*[t.data_ptr() for t in ts]))
            _lib.check(lib.mp_query_points_vjp_ex(
                mlp, fh.ptr, B, ctypes.c_void_p(p.data_ptr()), n, s[0], s[1], s[2],
                None if cal is None else ctypes.c_void_p(cal.data_ptr()), proj, ctypes.c_float(self.normalizer.scale),
                ctypes.c_void_p(gout.data_ptr()), None if dfeat is None else ctypes.c_void_p(dfeat.data_ptr()),
                None if dpoints is None else ctypes.c_void_p(dpoints.data_ptr()), ptrs(dws), ptrs(dbs),
                None if scratch is None else ctypes.c_void_p(scratch.data_ptr()), int(nbytes), flags, _lib.stream_ptr(dev)),
                "mp_query_points_vjp_ex")
        return dfeat, dpoints, dws, dbs

    def _query_batch(self, feat, points, calibs):
        """query() of B > 1 images: one launch; the calibs stay on the device (no read-back, no synchronisation)."""
        B = feat.shape[0]
        if points.dim() != 3 or points.shape[1] != 3 or points.shape[0] != B:
            raise ValueError("points must be [B,3,N] with the features' B=%d; got %s" % (B, tuple(points.shape)))
        if calibs is not None and (calibs.dim() != 3 or calibs.shape[0] != B or calibs.shape[1] not in (3, 4)
                                   or calibs.shape[2] != 4):
            raise ValueError("calibs must be [B,4,4] or [B,3,4] with the features' B=%d; got %s" % (B, tuple(calibs.shape)))
        if points.device != feat.device:
            raise ValueError("points and features live on different devices")
        if points.dtype != torch.float32:
            points = points.float()
        n = points.shape[2]
        s = points.stride()
        if n > 0 and min(s) < 1:
            points = points.contiguous()
            s = points.stride()
        res = self.surface_classifier.filter_channels[-1]
        out = torch.empty((B, res, n), dtype=torch.float32, device=feat.device)
        if n == 0:
            return [out]
        with _lib.device_guard(feat.device):
            cal = None
            if calibs is not None:
                cal = calibs.detach()[:, :3, :4].to(device=feat.device, dtype=torch.float32).contiguous()
            fh = self.batch_feature_handle(feat)
            proj = _lib.PROJ_PERSPECTIVE if self.projection is perspective else _lib.PROJ_ORTHOGONAL
            _lib.check(_lib.load().mp_query_points_batch(
                self.surface_classifier.handle(), fh.ptr, B, ctypes.c_void_p(points.data_ptr()), n, s[0], s[1], s[2],
                None if cal is None else ctypes.c_void_p(cal.data_ptr()), proj, ctypes.c_float(self.normalizer.scale),
                ctypes.c_void_p(out.data_ptr()), res * n, n, self._mode(), _lib.stream_ptr(feat.device)),
                "mp_query_points_batch")
        return [out]

    def query_grid(self, feat, calibs, resolution, b_min, b_max, z0=0, nz=None, out=None, fh=None):
        """Dense occupancy slab [nz,R,R] of an R^3 grid over [b_min,b_max] (points generated in-kernel).
        `fh`: a handle already uploaded for this frame (`feature_handle(feat)`), to skip the upload here."""
        R = int(resolution)
        nz = R - z0 if nz is None else int(nz)
        if out is None:
            out = torch.empty((nz, R, R), dtype=torch.float32, device=feat.device)
        with _lib.device_guard(feat.device):
            if fh is None:
                fh = self.feature_handle(feat)
            proj = _lib.PROJ_PERSPECTIVE if self.projection is perspective else _lib.PROJ_ORTHOGONAL
            _lib.check(_lib.load().mp_query_grid(
                self.surface_classifier.handle(), fh.ptr, R, int(z0), nz, _lib.f3(b_min), _lib.f3(b_max),
                _lib.calib12(calibs), proj, ctypes.c_float(self.normalizer.scale), ctypes.c_void_p(out.data_ptr()),
                self._mode(), _lib.stream_ptr(feat.device)), "mp_query_grid")
        return out

    def query_grid_range(self, feat, calibs, resolution, b_min, b_max, lin0, n, out=None, fh=None):
        """Occupancy of nodes [lin0, lin0+n) of the R^3 grid's z-major linear order (balanced multi-GPU sharding, see
        shard.range_bounds); `out` = a float32 CUDA buffer of at least n elements."""
        R, lin0, n = int(resolution), int(lin0), int(n)
        if out is None:
            out = torch.empty(n, dtype=torch.float32, device=feat.device)
        if n == 0:
            return out
        with _lib.device_guard(feat.device):
            if fh is None:
                fh = self.feature_handle(feat)
            proj = _lib.PROJ_PERSPECTIVE if self.projection is perspective else _lib.PROJ_ORTHOGONAL
            _lib.check(_lib.load().mp_query_grid_range(
                self.surface_classifier.handle(), fh.ptr, R, lin0, n, _lib.f3(b_min), _lib.f3(b_max),
                _lib.calib12(calibs), proj, ctypes.c_float(self.normalizer.scale), ctypes.c_void_p(out.data_ptr()),
                self._mode(), _lib.stream_ptr(feat.device)), "mp_query_grid_range")
        return out

    # ---- training scaffolding kept for API parity ---------------------------------------------------------
    def get_loss(self, pred_stages, labels):
        fn = {"MSE": F.mse_loss, "L1": F.l1_loss}.get(self.opt.loss.IMF)
        if fn is None:
            raise NotImplementedError
        return sum(fn(p, labels) for p in pred_stages) / len(pred_stages)

    def forward(self, images, points, calibs, transforms=None, labels=None, feat_prior=None):
        pred_stages = self.query(self.filter(images, feat_prior), points, calibs, transforms)
        if labels is not None:
            return pred_stages[-1], self.get_loss(pred_stages, labels)
        return pred_stages[-1]

    def load_legacy_pifu(self, ckpt_path):
        """Flat PIFu state dict: `surface_classifier.conv{i}.*` -> `filters.{i}.*` (MonoPortNet.py:153-160)."""
        ckpt = torch.load(ckpt_path, map_location="cpu")
        self.image_filter.load_state_dict(
            {k.replace("image_filter.", ""): v for k, v in ckpt.items() if "image_filter" in k})
        self.surface_classifier.load_state_dict(
            {k.replace("surface_classifier.conv", "filters."): v for k, v in ckpt.items() if "surface_classifier" in k})


def _opt(backbone, head, loss):
    o = CN()
    o.projection = "orthogonal"
    o.backbone = CN(); o.backbone.IMF = backbone
    o.normalizer = CN(); o.normalizer.IMF = 'PIFuNomalizer'
    o.head = CN(); o.head.IMF = head
    o.loss = CN(); o.loss.IMF = loss
    return o


def PIFuNetG():
    return MonoPortNet(_opt('PIFuHGFilters', 'PIFuNetGMLP', 'MSE'))


def PIFuNetC():
    return MonoPortNet(_opt('PIFuResBlkFilters', 'PIFuNetCMLP', 'L1'))
