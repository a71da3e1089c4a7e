"""Frame-stream overlap (SURVEY.md §8f-2).  The reference chains its per-frame stages as `processors=[callable, ...]`
with one Python thread per stage (RTL/dataloader.py:734-751, 1026-1054).  On one big GPU the useful overlap is between
FRAMES: frame k+1's encoder (PyTorch) can run while frame k's reconstruction kernels do.  `FramePipeline` keeps the
list-of-callables API, dispatches frames round-robin to `n_lanes` worker threads that each own a CUDA stream, and yields
results in order.  All monoport_b200 handles that carry per-call scratch are per-thread, so lanes do not share state."""
import ctypes
import threading
from collections import deque
from concurrent.futures import ThreadPoolExecutor

import torch

from . import _lib


class FramePipeline:
    def __init__(self, processors, device="cuda:0", n_lanes=2):
        self.processors = list(processors)
        self.device = torch.device(device)
        self.n_lanes = int(n_lanes)
        self._pool = ThreadPoolExecutor(max_workers=self.n_lanes, thread_name_prefix="mp_lane")
        self._tls = threading.local()

    def _run_one(self, item):
        if not hasattr(self._tls, "stream"):
            torch.cuda.set_device(self.device)                 # RTL/dataloader.py:1031
            self._tls.stream = torch.cuda.Stream(self.device)
        with torch.cuda.stream(self._tls.stream):
            data = item
            for p in self.processors:
                data = p(data)
            self._tls.stream.synchronize()
        return data

    def run(self, iterable):
        """Generator: results in input order, up to n_lanes frames in flight."""
        inflight = deque()
        for item in iterable:
            inflight.append(self._pool.submit(self._run_one, item))
            if len(inflight) >= self.n_lanes:
                yield inflight.popleft().result()
        while inflight:
            yield inflight.popleft().result()

    def close(self):
        self._pool.shutdown(wait=True)


class FrameGraph:
    """One frame = ONE CUDA-graph launch:  [image -> encoder (PyTorch) ->]  features -> coarse-to-fine engine -> visible surface.

    The reference overlaps its per-frame stages with one Python thread per stage (RTL/dataloader.py:734-751, 1026-1054) and
    pays a host round trip between every pair of them.  Here the whole frame step is captured once (the encoder's PyTorch
    kernels and this library's enqueue-only entry points mp_octree_run_fused_async / mp_forward_vertices_async on one
    stream) and replayed per frame: no Python, no launch gaps and no host synchronisation inside a frame -- even the choice
    between the tensor-core and the exact kernel is made on the device (range guard).  Several FrameGraphs own separate
    streams, workspaces and output buffers, so frame k+1's encoder overlaps frame k's reconstruction (`FrameGraphRing`).

    engine: a Seg3dLossless (faster=True, or the lossless faster=False) / Seg3dTopk built with make_query_func(net).  The
    lossless engine's conflict loop runs inside the graph as a conditional WHILE node per level, decided on the device;
    result() reads its passes per level into `last_conflict_loops` and raises RuntimeError for a frame whose loop stopped at
    its cap (8 x the level's resolution passes) -- run that frame with the eager engine.
    calib: [1,4,4] tensor, the graph's default camera.  The graph reads its camera from a 12-float device buffer when it runs
    (the _dcal entry points), so every frame can have its own: launch(x, calib=...) writes the frame's camera there before
    the replay, launch(x) the default one.  Orthographic or perspective projection stays the net's, fixed at construction.
    `feature_hook(feat) -> feat` (optional) runs inside the captured step on the encoder's last-stage map.
    launch(x) enqueues a frame (x = image [1,3,H,W] with an encoder, else the [1,C,h,w] feature map); result() waits for it
    and returns (sdf or None, X, Y, Z, norm) exactly like engine(..., calib_tensor=<the frame's camera>) followed by
    forward_vertices(sdf, direction).

    The demo's two images (RTL/main.py:417-441) can be rendered inside the same captured step:
      netC: the colour net.  Its map is netC.filter(x_colour, feat_prior=<the geometry map the engine receives>) with the
        encoder (MonoPortNet.py:41-45, RTL/main.py:373-379), else x_colour itself ([1,C,h,w]); netC is queried at the
        visible vertices into an [R,R,3] canvas like colorization(netC, ...) -- mp_colorize_surface_async: the vertex count
        stays on the device and the range guard of the tensor-core colour program is decided there (a frame outside it
        is rendered by the exact fp32 kernel, like netC.query would evaluate it);
      render_normals: the normal image, like colorization(norm=N) (mp_render_normals_async).  True: N = forward_vertices'
        finite-difference normals (the norm result() returns); "gradient": N = the analytic normals of the geometry net,
        surface_normals(..., precision="auto") computed inside the step (mp_surface_normals_async, the count on the device);
      canvas: the background of both images ([R,R,3], default ones).
    launch(x, x_colour) then takes the netC input too, and rendered() (after result()) returns (render_norm, render_tex).

    The mesh of the frame can be extracted inside the same captured step:
      mesh: marching cubes at 0.5 on the frame's volume, in world space (marching_cubes_async on a workspace the graph
        owns): the vertices and faces reconstruction(use_octree=True, engine=engine) returns for the frame, bit for bit;
      mesh_normals: their analytic normals, mesh_normals(net, ..., precision="auto") computed inside the step;
      mesh_colours: their colours, mesh_colours(netC, ...) computed inside the step (needs netC);
      mesh_capacity: (vertices, faces) the buffers hold, default (8 R^2, 16 R^2).
    mesh() (after result()) then returns (verts [V,3], faces [F,3] int32, normals or None, colours or None) -- views of this
    graph's buffers, valid until its next launch -- or None for a frame without a surface, and raises RuntimeError for a
    frame whose mesh exceeds the capacity (run reconstruction() eagerly for that frame).

    display: the step ends with the demo's display images (RTL/main.py:252-281) of the rendered images, copied into
      page-locked host buffers of this graph (mp_display_async; needs netC and/or render_normals).  displayed() (after
      result()) returns them as recon.visulization(*rendered()) does -- numpy views of those buffers, valid until the next
      launch -- with no device work of its own."""

    def __init__(self, net, engine, calib, direction="front", with_encoder=True, input_shape=None, feature_hook=None,
                 netC=None, render_normals=False, canvas=None, mesh=False, mesh_normals=False, mesh_colours=False,
                 mesh_capacity=None, display=False):
        from .modeling.MonoPortNet import FeatureHandle
        from .modeling.geometry import perspective
        from .recon import _DIRS
        if getattr(engine.query_func, "__monoport_fused__", None) is not net:
            raise ValueError("the engine's query_func must be make_query_func(net)")
        self.net, self.engine = net, engine
        dev = self.device = engine.b_min.device
        self.with_encoder = bool(with_encoder)
        self.feature_hook = feature_hook
        self.R = R = engine.resolutions[-1]
        self._dir = _DIRS[direction]
        self._proj = _lib.PROJ_PERSPECTIVE if net.projection is perspective else _lib.PROJ_ORTHOGONAL
        cal12 = _lib.calib12(calib.detach().cpu())
        if input_shape is None:
            input_shape = (1, 3, 512, 512) if with_encoder else (1, net.surface_classifier.filter_channels[0] - 1, 128, 128)
        self.netC = netC
        if render_normals not in (False, True, "gradient"):
            raise ValueError("render_normals must be False, True or 'gradient'; got %r" % (render_normals,))
        self.render_normals = render_normals
        if (mesh_normals or mesh_colours or mesh_capacity is not None) and not mesh:
            raise ValueError("mesh_normals, mesh_colours and mesh_capacity need mesh=True")
        if mesh_colours and netC is None:
            raise ValueError("mesh_colours needs netC")
        self.with_mesh, self.with_mesh_normals, self.with_mesh_colours = bool(mesh), bool(mesh_normals), bool(mesh_colours)
        if display and netC is None and not render_normals:
            raise ValueError("display needs an image to show: netC and/or render_normals")
        self.with_display = bool(display)
        lib = self._lib = _lib.load()
        with torch.cuda.device(dev):
            self.stream = torch.cuda.Stream(dev)
            self.static_in = torch.zeros(input_shape, dtype=torch.float32, device=dev)
            # the camera the captured step reads when it runs (rows 0..2 of [R|t]), and the constructor's, for launch(calib=None)
            self._cal_default = torch.tensor(list(cal12), dtype=torch.float32).to(dev)
            self._cal_dev = self._cal_default.clone()
            self._cal_is_default = True           # (only launch() writes the buffer, in stream order)
            self.render_tex = self.render_norm = None
            if netC is not None or self.render_normals:
                bg = torch.ones((R, R, 3), dtype=torch.float32) if canvas is None else canvas.detach()
                if tuple(bg.shape) != (R, R, 3):
                    raise ValueError("canvas must be [%d,%d,3] (the engine's resolution); got %s" % (R, R, tuple(bg.shape)))
                self._bg = bg.to(device=dev, dtype=torch.float32).contiguous()
                self.render_norm = torch.empty_like(self._bg) if self.render_normals else None
            if netC is not None:
                if with_encoder:                    # the netC image, the same size as the geometry net's
                    colour_shape = input_shape
                else:                               # netC's own map, at the geometry map's size
                    colour_shape = (1, netC.surface_classifier.filter_channels[0] - 1) + tuple(input_shape[2:])
                self.static_in_c = torch.zeros(colour_shape, dtype=torch.float32, device=dev)
                self.render_tex = torch.empty_like(self._bg)
                self._fhc = None
                self._headC = netC.surface_classifier.handle()
                self._projC = _lib.PROJ_PERSPECTIVE if netC.projection is perspective else _lib.PROJ_ORTHOGONAL
            self._bmin3, self._bmax3 = _lib.f3(engine.b_min), _lib.f3(engine.b_max)
            self.volume = torch.empty((1, 1, R, R, R), dtype=torch.float32, device=dev)
            cap = R * R
            self.X = torch.empty(cap, dtype=torch.int64, device=dev)
            self.Y = torch.empty(cap, dtype=torch.int64, device=dev)
            self.Z = torch.empty(cap, dtype=torch.float32, device=dev)
            self.N = torch.empty((cap, 3), dtype=torch.float32, device=dev)
            self.count = torch.zeros(1, dtype=torch.int64, device=dev)
            if render_normals == "gradient":
                self.N_grad = torch.empty((cap, 3), dtype=torch.float32, device=dev)
                self._nscratch = torch.empty(6 * cap + 1, dtype=torch.float32, device=dev)
            self._scratch = torch.empty(int(lib.mp_forward_vertices_scratch_bytes(R)), dtype=torch.uint8, device=dev)
            self._mcubes = None
            if mesh:
                from .recon import McubesWorkspace
                v_cap, f_cap = (8 * R * R, 16 * R * R) if mesh_capacity is None else (int(c) for c in mesh_capacity)
                if v_cap < 0 or f_cap < 0:
                    raise ValueError("mesh_capacity must be (vertices, faces) >= 0; got %r" % (mesh_capacity,))
                self._mcubes = McubesWorkspace((R, R, R), dev)
                self.mesh_verts = torch.empty((v_cap, 3), dtype=torch.float32, device=dev)
                self.mesh_faces = torch.empty((f_cap, 3), dtype=torch.int32, device=dev)
                self.mesh_counts = torch.zeros(2, dtype=torch.int64, device=dev)
                self._mesh_count32 = torch.zeros(1, dtype=torch.int32, device=dev)
                if mesh_normals:
                    self.mesh_norm = torch.empty((v_cap, 3), dtype=torch.float32, device=dev)
                    self._mesh_nscratch = torch.empty(3 * v_cap, dtype=torch.float32, device=dev)
                if mesh_colours:
                    self._mesh_pred = torch.empty((3, v_cap), dtype=torch.float32, device=dev)
                    self._mesh_rgb = torch.empty((3, v_cap), dtype=torch.float32, device=dev)
            if display:
                from .recon import DisplayBuffers
                self._display = DisplayBuffers(self.render_norm is not None, self.render_tex is not None, dev)
            self._oct = engine._new_handle(dev)            # private workspace: graphs of different lanes overlap
            self._fh = None
            self._head = net.surface_classifier.handle()
            self._FeatureHandle = FeatureHandle
            # eager warm-up on the side stream (lazy allocations, cudnn autotune), then the capture
            self.stream.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(self.stream), torch.no_grad():
                for _ in range(2):
                    self._step()
            self.stream.synchronize()
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph, stream=self.stream), torch.no_grad():
                self._step()
        self.last_stats = None
        self.last_conflict_loops = None
        self._nonempty = None

    def _step(self):
        lib, dev = self._lib, self.device
        if self.with_encoder:
            feat = self.net.filter(self.static_in)[-1][0]
        else:
            feat = self.static_in
        if self.feature_hook is not None:
            feat = self.feature_hook(feat)
        if self._fh is None:
            _, C, H, W = feat.shape
            self._fh = self._FeatureHandle(C, H, W, dev)
        self._fh.key = None                      # always upload: the map changes with every replay
        self._fh.upload(feat)
        st = _lib.stream_ptr(dev)
        cal = ctypes.c_void_p(self._cal_dev.data_ptr())
        _lib.check(lib.mp_octree_run_fused_async_dcal(
            self._oct, self._head, self._fh.ptr, cal, self._proj, ctypes.c_float(self.net.normalizer.scale),
            self.net._mode(), ctypes.c_void_p(self.volume.data_ptr()), st), "mp_octree_run_fused_async_dcal")
        _lib.check(lib.mp_forward_vertices_async(
            ctypes.c_void_p(self.volume.data_ptr()), self.R, self._dir, ctypes.c_void_p(self.X.data_ptr()),
            ctypes.c_void_p(self.Y.data_ptr()), ctypes.c_void_p(self.Z.data_ptr()), ctypes.c_void_p(self.N.data_ptr()),
            ctypes.c_void_p(self.count.data_ptr()), ctypes.c_void_p(self._scratch.data_ptr()), st), "mp_forward_vertices_async")
        cap = self.X.numel()
        if self.render_normals:
            norm = self.N
            if self.render_normals == "gradient":
                norm = self.N_grad
                _lib.check(lib.mp_surface_normals_async_dcal(
                    self._head, self._fh.ptr, ctypes.c_void_p(self.X.data_ptr()), ctypes.c_void_p(self.Y.data_ptr()),
                    ctypes.c_void_p(self.Z.data_ptr()), ctypes.c_void_p(self.count.data_ptr()), cap, self.R, self._bmin3,
                    self._bmax3, cal, self._proj, ctypes.c_float(self.net.normalizer.scale), _lib.MODE_AUTO,
                    ctypes.c_void_p(self._nscratch.data_ptr()), ctypes.c_void_p(norm.data_ptr()), st),
                    "mp_surface_normals_async_dcal")
            self.render_norm.copy_(self._bg)
            _lib.check(lib.mp_render_normals_async(
                ctypes.c_void_p(self.X.data_ptr()), ctypes.c_void_p(self.Y.data_ptr()), ctypes.c_void_p(norm.data_ptr()),
                ctypes.c_void_p(self.count.data_ptr()), cap, self.R, ctypes.c_void_p(self.render_norm.data_ptr()), st),
                "mp_render_normals_async")
        if self.netC is not None:
            # netC's map: its encoder with the geometry map the engine received as the prior, or the map as given
            featc = self.netC.filter(self.static_in_c, feat_prior=feat)[-1][0] if self.with_encoder else self.static_in_c
            if self._fhc is None:
                _, C, H, W = featc.shape
                self._fhc = self._FeatureHandle(C, H, W, dev)
            self._fhc.key = None
            self._fhc.upload(featc)
            self.render_tex.copy_(self._bg)
            _lib.check(lib.mp_colorize_surface_async_dcal(
                self._headC, self._fhc.ptr, ctypes.c_void_p(self.X.data_ptr()), ctypes.c_void_p(self.Y.data_ptr()),
                ctypes.c_void_p(self.Z.data_ptr()), ctypes.c_void_p(self.count.data_ptr()), cap, self.R, self._bmin3,
                self._bmax3, cal, self._projC, ctypes.c_float(self.netC.normalizer.scale), self.netC._mode(),
                ctypes.c_void_p(self.render_tex.data_ptr()), st), "mp_colorize_surface_async_dcal")
        if self.with_mesh:
            self._mesh_step(st, cal)
        if self.with_display:
            self._display.enqueue(self.render_norm, self.render_tex, self.R, st)

    def _mesh_step(self, st, cal):
        from .recon import marching_cubes_async
        lib = self._lib
        marching_cubes_async(self.volume, self.mesh_verts, self.mesh_faces, self.mesh_counts, self._mesh_count32, 0.5,
                             list(self._bmin3), list(self._bmax3), workspace=self._mcubes)
        v_cap = self.mesh_verts.shape[0]
        verts, counts, count32 = (ctypes.c_void_p(t.data_ptr()) for t in (self.mesh_verts, self.mesh_counts, self._mesh_count32))
        if self.with_mesh_normals:
            _lib.check(lib.mp_mesh_normals_async_dcal(
                self._head, self._fh.ptr, verts, counts, count32, v_cap, cal, self._proj,
                ctypes.c_float(self.net.normalizer.scale), _lib.MODE_AUTO, ctypes.c_void_p(self._mesh_nscratch.data_ptr()),
                ctypes.c_void_p(self.mesh_norm.data_ptr()), st), "mp_mesh_normals_async_dcal")
        if self.with_mesh_colours:
            # netC at the vertex rows (row stride 1, point stride 3), then mesh_colours' pred * 0.5 + 0.5
            _lib.check(lib.mp_query_points_count_dcal(
                self._headC, self._fhc.ptr, verts, v_cap, 1, 3, cal, self._projC,
                ctypes.c_float(self.netC.normalizer.scale), ctypes.c_void_p(self._mesh_pred.data_ptr()), v_cap, count32,
                self.netC._mode(), st), "mp_query_points_count_dcal")
            torch.mul(self._mesh_pred, 0.5, out=self._mesh_rgb)
            self._mesh_rgb.add_(0.5)

    def _calib_rows(self, calib):
        """calib ([1,4,4], [4,4] or [3,4], any float dtype, on the CPU or on the graph's device) -> its rows 0..2 as a
        [3,4] tensor, the reduction of _lib.calib12 (the float32 rounding happens in the copy into the buffer)."""
        if not torch.is_tensor(calib) or not calib.is_floating_point():
            raise ValueError("calib must be a floating-point tensor; got %r" % (type(calib) if not torch.is_tensor(calib)
                                                                               else calib.dtype,))
        c = calib.detach()
        if c.dim() == 3:
            if c.shape[0] != 1:
                raise ValueError("calib: batch size must be 1; got %d" % c.shape[0])
            c = c[0]
        if c.dim() != 2 or c.shape[1] != 4 or c.shape[0] not in (3, 4):
            raise ValueError("calib must be [1,4,4], [4,4] or [3,4]; got %s" % (tuple(calib.shape),))
        if c.device.type != "cpu" and c.device != self._cal_dev.device:
            raise ValueError("calib is on %s; the FrameGraph runs on %s (or pass a CPU tensor)" % (c.device, self._cal_dev.device))
        if c.device.type == "cpu":
            # a private copy: the caller may change its tensor as soon as launch() returns
            c = c[:3, :4].to(torch.float32, copy=True)
        return c[:3, :4]

    def launch(self, x, x_colour=None, calib=None):
        """Enqueue one frame (returns at once).  x_colour: netC's input (its image with the encoder, else its map), required
        exactly when the graph was built with netC.  calib: the frame's camera ([1,4,4], [4,4] or [3,4], CPU or this graph's
        device; rows 0..2 are used, in float32 like calib12), None for the constructor's.  ValueError for another shape, a
        batch of more than one or another device."""
        if (x_colour is None) != (self.netC is None):
            raise ValueError("x_colour is required exactly when the FrameGraph renders with netC")
        rows = None if calib is None else self._calib_rows(calib)
        self.stream.wait_stream(torch.cuda.current_stream(self.device))     # x may still be produced on the caller's stream
        with torch.cuda.stream(self.stream):
            if rows is None:
                if not self._cal_is_default:      # a fixed camera costs nothing per frame
                    self._cal_dev.copy_(self._cal_default, non_blocking=True)
                    self._cal_is_default = True
            else:
                self._cal_is_default = False
                if rows.device.type != "cpu":
                    rows.record_stream(self.stream)      # (read on this stream: its memory is not reused before the copy)
                self._cal_dev.view(3, 4).copy_(rows, non_blocking=True)
            self.static_in.copy_(x, non_blocking=True)
            if x_colour is not None:
                self.static_in_c.copy_(x_colour, non_blocking=True)
            self.graph.replay()
        self._nonempty = None
        return self

    def result(self):
        """Wait for the enqueued frame: (sdf or None, X, Y, Z, norm) -- views of this graph's buffers, valid until its next launch.
        Raises RuntimeError when the lossless conflict loop of the frame stopped at its cap."""
        n = len(self.engine.resolutions)
        nonempty = ctypes.c_int(0)
        stats = (ctypes.c_int64 * n)()
        loops = (ctypes.c_int32 * n)()
        with torch.cuda.stream(self.stream):
            st = _lib.stream_ptr(self.device)
            _lib.check(self._lib.mp_octree_fetch(self._oct, ctypes.byref(nonempty), stats, st),
                       "mp_octree_fetch")                                    # (synchronises the graph's stream)
            rc = self._lib.mp_octree_fetch_loops(self._oct, loops, st)
        self.last_stats = list(stats)
        self.last_conflict_loops = list(loops)
        if rc == _lib.MP_E_TRUNCATED:
            self._nonempty = None
            raise RuntimeError("FrameGraph: %s; this frame's volume is incomplete -- run the eager engine for it"
                               % self._lib.mp_last_error().decode())
        _lib.check(rc, "mp_octree_fetch_loops")
        self._nonempty = bool(nonempty.value)
        if not nonempty.value:
            return None, None, None, None, None
        k = int(self.count.item())
        return self.volume, self.X[:k], self.Y[:k], self.Z[:k], self.N[:k]

    def rendered(self):
        """After result(): (render_norm, render_tex), the [R,R,3] images of the frame -- views of this graph's buffers, valid
        until its next launch.  An image the graph was not built to render is None; both are None for an empty frame (like
        colorization(X=None))."""
        if self._nonempty is None:
            raise RuntimeError("FrameGraph.rendered() needs the frame's result() first")
        if not self._nonempty:
            return None, None
        return self.render_norm, self.render_tex

    def mesh(self):
        """After result(): (verts [V,3] world, faces [F,3] int32, normals [V,3] or None, colours [V,3] or None) of the frame
        -- views of this graph's buffers, valid until its next launch -- or None when the frame has no surface.  Raises
        RuntimeError when the frame's mesh does not fit the graph's capacity."""
        if not self.with_mesh:
            raise RuntimeError("FrameGraph.mesh() needs a graph built with mesh=True")
        if self._nonempty is None:
            raise RuntimeError("FrameGraph.mesh() needs the frame's result() first")
        if not self._nonempty:
            return None
        nv, nf = self.mesh_counts.tolist()              # (result() has synchronised the graph's stream)
        v_cap, f_cap = self.mesh_verts.shape[0], self.mesh_faces.shape[0]
        if nv > v_cap or nf > f_cap:
            raise RuntimeError("FrameGraph: the frame's mesh has %d vertices and %d faces, above the capacity of %d and %d "
                               "(mesh_capacity) -- run reconstruction() eagerly for this frame" % (nv, nf, v_cap, f_cap))
        if nv == 0:
            return None
        return (self.mesh_verts[:nv], self.mesh_faces[:nf], self.mesh_norm[:nv] if self.with_mesh_normals else None,
                self._mesh_rgb.t()[:nv] if self.with_mesh_colours else None)

    def displayed(self):
        """After result(): (render_norm [256,256,3] float32, render_tex likewise, mask [256,256,1] bool) -- numpy views of
        this graph's page-locked buffers, valid until its next launch, equal to recon.visulization(*rendered()).  An image
        the graph does not render is None; all three are None for an empty frame."""
        if not self.with_display:
            raise RuntimeError("FrameGraph.displayed() needs a graph built with display=True")
        if self._nonempty is None:
            raise RuntimeError("FrameGraph.displayed() needs the frame's result() first")
        if not self._nonempty:
            return None, None, None
        return self._display.arrays

    def close(self):
        if self._oct is not None:
            self.stream.synchronize()
            self._lib.mp_octree_destroy(self._oct)
            self._oct = None
        if self._mcubes is not None:
            self.stream.synchronize()
            self._mcubes.close()
            self._mcubes = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class FrameGraphRing:
    """`n_lanes` FrameGraphs used round-robin: up to n_lanes frames in flight, results in input order (the graph-captured
    counterpart of FramePipeline for the stages of this library).  Lanes built with netC take (x, x_colour) items and yield
    result() + rendered(): (sdf, X, Y, Z, norm, render_norm, render_tex).  Lanes built with mesh=True append mesh()'s
    (verts, faces, normals, colours), four Nones for a frame without a surface.  Lanes built with display=True then append
    displayed()'s (render_norm, render_tex, mask).  run(items, calibs) takes the cameras of the frames too (zipped with
    items; see FrameGraph.launch)."""

    def __init__(self, make_graph, n_lanes=2):
        self.lanes = [make_graph() for _ in range(int(n_lanes))]

    @staticmethod
    def _out(lane):
        out = lane.result()
        if lane.netC is not None or lane.render_normals:
            out = out + lane.rendered()
        if lane.with_mesh:
            out = out + (lane.mesh() or (None,) * 4)
        if lane.with_display:
            out = out + lane.displayed()
        return out

    def run(self, iterable, calibs=None):
        inflight = deque()
        pairs = zip(iterable, calibs) if calibs is not None else ((x, None) for x in iterable)
        for i, (x, calib) in enumerate(pairs):
            lane = self.lanes[i % len(self.lanes)]
            if len(inflight) >= len(self.lanes):
                yield self._out(inflight.popleft())
            inflight.append(lane.launch(*x, calib=calib) if lane.netC is not None else lane.launch(x, calib=calib))
        while inflight:
            yield self._out(inflight.popleft())

    def close(self):
        for lane in self.lanes:
            lane.close()
