"""Coarse-to-fine occupancy engines with the call-site contract of `implicit_seg.functional`
(third-party, un-vendored in the reference: requirements.txt:15; ctor RTL/main.py:188-195, call :390-395,
result consumer RTL/recon.py:32-38).  PARITY UNPINNED against upstream (see DESIGN.md).

All index/byte work (2x up-sampling, boundary+dilation, ordered compaction, scatter, conflict loop, top-k select)
runs in the sm_90a kernels of csrc/octree.cu through the C-ABI.  Two drive modes, identical volumes:
  * generic : any Python `query_func(points=[1,N,3], **kwargs) -> [1,1,N]` is called back once per batch
              (stepping API: mp_octree_begin / next / commit / finish);
  * fused   : when `query_func` was built by `make_query_func(net)` (it then carries `__monoport_fused__`),
              the whole pyramid runs on the device with the fused sample+MLP kernel and a single host sync
              at the end (mp_octree_run_fused).
"""
import ctypes
import threading

import numpy as np
import torch
import torch.nn as nn

from .. import _lib


def make_query_func(net):
    """The closure of RTL/main.py:168-183 around `net.query`, tagged so the engines can take the fused path."""

    @torch.no_grad()
    def query_func(points, im_feat_list, calib_tensor):
        assert len(points) == 1                                   # RTL/main.py:175
        samples = points.permute(0, 2, 1)                         # [1,3,N] view, no copy
        return net.query(im_feat_list, points=samples, calibs=calib_tensor)[0]

    query_func.__monoport_fused__ = net
    return query_func


def _as3(v):
    a = np.asarray(v.detach().cpu() if hasattr(v, "detach") else v, dtype=np.float32).reshape(-1)
    assert a.size == 3, "b_min / b_max must hold 3 values"
    return a


class _Seg3dBase(nn.Module):
    def __init__(self, query_func, b_min, b_max, resolutions, balance_value, faster, topk_points):
        super().__init__()
        self.query_func = query_func
        res = [int(r[0]) if hasattr(r, "__len__") else int(r) for r in resolutions]
        for r in res:
            assert r % 2 == 1, "resolution {} need to be odd because of align_corner.".format(r)
        self.resolutions = res
        self.balance_value = float(balance_value)
        self.faster = bool(faster)
        self.topk_points = None if topk_points is None else [0 if p is None else int(p) for p in topk_points]
        self.register_buffer("b_min", torch.from_numpy(_as3(b_min)).view(1, 1, 3))
        self.register_buffer("b_max", torch.from_numpy(_as3(b_max)).view(1, 1, 3))
        self._handles = {}
        self._mapped = []
        self._sharded = None
        self.last_stats = None

    def __getstate__(self):          # engine workspaces / peer mappings are native and per-thread: a copy starts without them
        d = dict(self.__dict__)
        d["_handles"], d["_mapped"], d["_sharded"] = {}, [], None
        return d

    def _new_handle(self, device):
        """A fresh engine workspace (mp_octree_t) with this engine's parameters."""
        n = len(self.resolutions)
        res = (ctypes.c_int * n)(*self.resolutions)
        topk = None if self.topk_points is None else (ctypes.c_int * n)(*self.topk_points)
        h = ctypes.c_void_p()
        with _lib.device_guard(device):
            _lib.check(_lib.load().mp_octree_create(
                n, res, _lib.f3(self.b_min), _lib.f3(self.b_max), ctypes.c_float(self.balance_value),
                1 if self.faster else 0, topk, ctypes.byref(h)), "mp_octree_create")
        return h

    # one engine workspace per (device, calling thread)
    def _handle(self, device):
        key = (device.index if device.index is not None else torch.cuda.current_device(), threading.get_ident())
        h = self._handles.get(key)
        if h is None:
            h = self._handles[key] = self._new_handle(device)
        return h

    def __del__(self):
        try:
            self.unshard()
            for h in self._handles.values():
                _lib.load().mp_octree_destroy(h)
        except Exception:
            pass

    # ---- multi-GPU list sharding (SURVEY.md §8e) ------------------------------------------------------------
    def shard(self, rank, world_size, group=None):
        """Collective: split the MLP evaluations of every level's node list over the ranks of `group` (one process per
        GPU of one node).  Every rank keeps the whole pyramid (the volume passes are replicated: identical inputs give
        identical node lists, the lossless conflict loop included), evaluates its window of each list, and the fused
        kernel stores the values into all ranks' value lists over NVLink peer memory.  Afterwards every rank calls the
        engine with the same features / calib and receives the full volume, bit-identical to the single-GPU volume.
        Applies to the calling thread's workspace and to the fused drive mode (`make_query_func(net)`)."""
        import torch.distributed as dist
        lib = _lib.load()
        device = self.b_min.device
        if device.type != "cuda":
            raise RuntimeError("call .to('cuda:N') before shard()")
        self.unshard()
        h = self._handle(device)
        if world_size == 1:
            return self
        with _lib.device_guard(device):
            blob = ctypes.create_string_buffer(192)
            _lib.check(lib.mp_octree_shard_export(h, blob), "mp_octree_shard_export")
            blobs = [None] * world_size
            dist.all_gather_object(blobs, blob.raw, group=group)
            arrs = [(ctypes.c_void_p * world_size)() for _ in range(3)]
            for r in range(world_size):
                if r == rank:
                    continue
                for k in range(3):
                    p = ctypes.c_void_p()
                    _lib.check(lib.mp_ipc_open(blobs[r][64 * k:64 * (k + 1)], ctypes.byref(p)), "mp_ipc_open")
                    self._mapped.append(p)
                    arrs[k][r] = p.value
            _lib.check(lib.mp_octree_shard_set(h, int(rank), int(world_size), arrs[0], arrs[1], arrs[2]), "mp_octree_shard_set")
        self._sharded = (int(rank), int(world_size))
        if group is not None or dist.is_initialized():
            dist.barrier(group=group)        # nobody starts storing into a peer before every mapping exists
        return self

    def unshard(self):
        for p in getattr(self, "_mapped", []):
            _lib.load().mp_ipc_close(p)
        self._mapped = []
        if getattr(self, "_sharded", None):
            for h in self._handles.values():
                _lib.load().mp_octree_shard_set(h, 0, 1, None, None, None)
        self._sharded = None

    @torch.no_grad()
    def forward(self, **kwargs):
        device = self.b_min.device
        if device.type != "cuda":
            raise RuntimeError("monoport_b200 engines run on CUDA only (call .to('cuda:0') like RTL/main.py:195)")
        net = getattr(self.query_func, "__monoport_fused__", None)
        # one engine call = one frame: its per-level queries may reuse the frame's uploaded features / calib
        with _lib.frame_scope():
            if net is not None and set(kwargs) == {"im_feat_list", "calib_tensor"}:
                return self._forward_fused(net, device, **kwargs)
            return self._forward_generic(device, **kwargs)

    def _new_volume(self, device):
        R = self.resolutions[-1]
        return torch.empty((1, 1, R, R, R), dtype=torch.float32, device=device)

    def _forward_fused(self, net, device, im_feat_list, calib_tensor):
        lib = _lib.load()
        feat = im_feat_list[-1][0]
        if feat.device != device:
            raise ValueError("features on %s but the engine lives on %s" % (feat.device, device))
        out = self._new_volume(device)
        nonempty = ctypes.c_int(0)
        stats = (ctypes.c_int64 * len(self.resolutions))()
        with _lib.device_guard(device):
            fh = net.feature_handle(feat)
            _lib.check(lib.mp_octree_run_fused(
                self._handle(device), net.surface_classifier.handle(), fh.ptr, _lib.calib12(calib_tensor), net._proj(),
                ctypes.c_float(net.normalizer.scale), net._mode(), ctypes.c_void_p(out.data_ptr()),
                ctypes.byref(nonempty), stats, _lib.stream_ptr(device)), "mp_octree_run_fused")
        self.last_stats = list(stats)
        return out if nonempty.value else None

    def _forward_generic(self, device, **kwargs):
        if self._sharded:
            raise RuntimeError("a sharded engine needs the fused drive mode: query_func = make_query_func(net), called "
                               "with im_feat_list= and calib_tensor=")
        lib = _lib.load()
        h = self._handle(device)
        stats = [0] * len(self.resolutions)
        with _lib.device_guard(device):
            st = _lib.stream_ptr(device)
            _lib.check(lib.mp_octree_begin(h, st), "mp_octree_begin")
            while True:
                n = ctypes.c_int64(0)
                level = ctypes.c_int(0)
                pts_ptr, idx_ptr = ctypes.c_void_p(), ctypes.c_void_p()
                _lib.check(lib.mp_octree_next(h, ctypes.byref(n), ctypes.byref(level), ctypes.byref(pts_ptr),
                                              ctypes.byref(idx_ptr), st), "mp_octree_next")
                if n.value == 0:
                    break
                stats[level.value] += n.value
                points = _wrap_device_f32(pts_ptr.value, (1, n.value, 3), device)
                occ = self.query_func(**kwargs, points=points)               # [1,1,N]
                if occ.dim() != 3 or occ.shape[0] != 1 or occ.shape[1] != 1 or occ.shape[2] != n.value:
                    raise ValueError("query_func must return [1,1,N]; got %s" % (tuple(occ.shape),))
                occ = occ.to(device=device, dtype=torch.float32).contiguous()
                _lib.check(lib.mp_octree_commit(h, ctypes.c_void_p(occ.data_ptr()), st), "mp_octree_commit")
            out = self._new_volume(device)
            nonempty = ctypes.c_int(0)
            _lib.check(lib.mp_octree_finish(h, ctypes.c_void_p(out.data_ptr()), ctypes.byref(nonempty), st),
                       "mp_octree_finish")
        self.last_stats = stats
        return out if nonempty.value else None


def _wrap_device_f32(ptr, shape, device):
    """Zero-copy torch view of library-owned device memory (valid until the next engine call)."""
    n = int(np.prod(shape))

    class _Buf:
        pass

    b = _Buf()
    b.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f4", "data": (int(ptr), False), "version": 2}
    return torch.as_tensor(b, device=device).view(*shape)


class Seg3dLossless(_Seg3dBase):
    """`Seg3dLossless(query_func, b_min, b_max, resolutions, balance_value=0.5, use_cuda_impl=..., faster=...)`
    -- constructor keywords as used at RTL/main.py:188-195.  `use_cuda_impl`/`visualize`/`debug` are accepted
    for signature compatibility and ignored (everything here is CUDA)."""

    def __init__(self, query_func, b_min, b_max, resolutions, channels=1, balance_value=0.5, align_corners=False,
                 visualize=False, debug=False, use_cuda_impl=False, faster=False, use_shadow=False, **kwargs):
        if channels != 1:
            raise NotImplementedError("channels must be 1")
        if align_corners:
            raise NotImplementedError("align_corners=True point mapping is not supported")
        if use_shadow:
            raise NotImplementedError("use_shadow pruning is not supported")
        super().__init__(query_func, b_min, b_max, resolutions, balance_value, faster, None)


class Seg3dTopk(_Seg3dBase):
    """Top-k variant: per level evaluate the `num_points[l]` nodes closest to the balance value."""

    def __init__(self, query_func, b_min, b_max, resolutions, num_points, channels=1, balance_value=0.5,
                 align_corners=False, visualize=False, debug=False, use_cuda_impl=False, **kwargs):
        if channels != 1:
            raise NotImplementedError("channels must be 1")
        if align_corners:
            raise NotImplementedError("align_corners=True point mapping is not supported")
        assert len(num_points) == len(resolutions), "num_points needs one entry per resolution"
        super().__init__(query_func, b_min, b_max, resolutions, balance_value, False, num_points)


def plot_mask3D(*args, **kwargs):
    """implicit_seg.functional.utils.plot_mask3D is an interactive vtkplotter viewer (RTL/main.py:29,397-398,
    commented out at the call site).  Visualisation is out of scope."""
    raise NotImplementedError("plot_mask3D (interactive 3D viewer) is out of scope")
