"""Surface extraction + mesh reconstruction on the device.

  pifu_calib, forward_vertices : same signatures/returns as RTL/recon.py:4-25 / :27-89 (the reference file itself can
                                 also be used unchanged on the volumes the engines return);
  marching_cubes, reconstruction: additions asked for by the north star (the reference has no marching cubes;
                                 `reconstruction` follows upstream PIFu's signature);
  marching_cubes_async, mesh_normals, mesh_colours: the mesh of a captured frame (FrameGraph(mesh=True)) and its eager
                                 twins -- normals and upstream PIFu's gen_mesh_color vertex colours at the vertices;
  refine_mesh_async            : its vertices moved along their edges onto the network's own iso-surface
                                 (FrameGraph(mesh_refine=K), reconstruction(refine=K));
  visulization                 : the demo's display images (RTL/main.py:252-281), the eager twin of
                                 FrameGraph(display=True);
  render_mesh                  : the mesh drawn from viewer cameras by the reference GL renderer's normal and colour
                                 programs (DESIGN.md §F3.2), the eager twin of FrameGraph(views=...).
"""
import ctypes
import threading

import numpy as np
import torch

from . import _lib

_DIRS = {"front": 0, "back": 1, "left": 2, "right": 3}


@torch.no_grad()
def pifu_calib(extrinsic, intrinsic, device="cuda:0"):
    """inv(K' E' diag(1,-1,1,1)) in float64 -> float32 [1,4,4]  (RTL/recon.py:4-25; host-side, negligible)."""
    K = np.array(intrinsic, dtype=np.float64, copy=True)
    E = np.array(extrinsic, dtype=np.float64, copy=True)
    K[2, 2] = K[0, 0]
    K[2, 3] = 0
    E[2, 3] = 0
    m = np.linalg.inv(K @ E @ np.diag([1.0, -1.0, 1.0, 1.0]))
    return torch.from_numpy(m).unsqueeze(0).float().to(device)


@torch.no_grad()
def forward_vertices(sdf, direction="front"):
    """Visible-surface vertices + normals of a [1,1,R,R,R] occupancy volume (RTL/recon.py:27-89), one kernel pass."""
    if sdf is None:
        return None, None, None, None
    if sdf.device.type != "cuda":
        raise RuntimeError("monoport_b200.forward_vertices: CUDA tensors only (no CPU path)")
    vol = sdf[0, 0]
    if vol.dtype != torch.float32 or not vol.is_contiguous():
        vol = vol.float().contiguous()
    R = vol.shape[2]
    assert vol.shape[0] == R and vol.shape[1] == R, "cubic volumes only"
    dev = vol.device
    cap = R * R
    X = torch.empty(cap, dtype=torch.int64, device=dev)
    Y = torch.empty(cap, dtype=torch.int64, device=dev)
    Z = torch.empty(cap, dtype=torch.float32, device=dev)
    N = torch.empty((cap, 3), dtype=torch.float32, device=dev)
    n = ctypes.c_int64(0)
    with _lib.device_guard(dev):
        _lib.check(_lib.load().mp_forward_vertices(
            ctypes.c_void_p(vol.data_ptr()), R, _DIRS[direction], ctypes.c_void_p(X.data_ptr()),
            ctypes.c_void_p(Y.data_ptr()), ctypes.c_void_p(Z.data_ptr()), ctypes.c_void_p(N.data_ptr()),
            ctypes.byref(n), _lib.stream_ptr(dev)), "mp_forward_vertices")
    k = n.value
    return X[:k], Y[:k], Z[:k], N[:k]


class _McubesWorkspace:
    _cache = {}

    @classmethod
    def get(cls, shape, device):
        key = (tuple(shape), device.index, threading.get_ident())
        h = cls._cache.get(key)
        if h is None:
            h = ctypes.c_void_p()
            with _lib.device_guard(device):
                _lib.check(_lib.load().mp_mcubes_create(shape[0], shape[1], shape[2], ctypes.byref(h)), "mp_mcubes_create")
            cls._cache[key] = h
        return h


@torch.no_grad()
def marching_cubes(vol, iso=0.5):
    """[D,H,W] (z,y,x) float32 CUDA volume -> (verts [V,3] float32 in index space (x,y,z), faces [F,3] int32).
    Indexed, watertight, deterministic ordering (see csrc/mcubes.cu)."""
    if vol.device.type != "cuda":
        raise RuntimeError("monoport_b200.marching_cubes: CUDA tensors only (no CPU path)")
    if vol.dim() == 5:
        vol = vol[0, 0]
    if vol.dtype != torch.float32 or not vol.is_contiguous():
        vol = vol.float().contiguous()
    dev = vol.device
    lib = _lib.load()
    h = _McubesWorkspace.get(vol.shape, dev)
    nv, nf = ctypes.c_int64(0), ctypes.c_int64(0)
    with _lib.device_guard(dev):
        st = _lib.stream_ptr(dev)
        _lib.check(lib.mp_mcubes_count(h, ctypes.c_void_p(vol.data_ptr()), ctypes.c_float(iso), ctypes.byref(nv),
                                       ctypes.byref(nf), st), "mp_mcubes_count")
        verts = torch.empty((nv.value, 3), dtype=torch.float32, device=dev)
        faces = torch.empty((nf.value, 3), dtype=torch.int32, device=dev)
        _lib.check(lib.mp_mcubes_emit(h, ctypes.c_void_p(vol.data_ptr()), ctypes.c_float(iso),
                                      ctypes.c_void_p(verts.data_ptr()), ctypes.c_void_p(faces.data_ptr()), st),
                   "mp_mcubes_emit")
    return verts, faces


class McubesWorkspace:
    """A marching-cubes workspace (mp_mcubes_t) for volumes of one [D,H,W] shape, owned by the caller: what
    marching_cubes_async runs on.  Runs that may be in flight together (the lanes of a FrameGraphRing, which share a thread)
    need one workspace each.  close() frees it once the work enqueued on it has completed."""

    def __init__(self, shape, device):
        self.shape = tuple(int(s) for s in shape)
        self.device = torch.device(device)
        self.ptr = ctypes.c_void_p()
        with _lib.device_guard(self.device):
            _lib.check(_lib.load().mp_mcubes_create(*self.shape, ctypes.byref(self.ptr)), "mp_mcubes_create")

    def close(self):
        if self.ptr:
            _lib.load().mp_mcubes_destroy(self.ptr)
            self.ptr = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _require(t, dtype, shape, what):
    if t.dtype != dtype or t.device.type != "cuda" or not t.is_contiguous() or (shape is not None and tuple(t.shape) != shape):
        raise ValueError("%s must be a contiguous %s CUDA tensor%s; got %s %s %s" % (
            what, dtype, "" if shape is None else " of shape %s" % (shape,), t.dtype, t.device, tuple(t.shape)))


@torch.no_grad()
def marching_cubes_async(vol, verts, faces, counts, count32, iso=0.5, b_min=None, b_max=None, *, workspace):
    """marching_cubes() without the host: enqueue-only (no read-back, no allocation, no synchronisation), so a CUDA graph
    can capture it (FrameGraph(mesh=True)).  The mesh goes into the caller's buffers verts [V_cap,3] float32 and faces
    [F_cap,3] int32 -- the same ids and order as marching_cubes(); vertices with id >= V_cap and faces with index >= F_cap are
    not written.  counts (int64 [2]) receives the true totals (nV, nF): the mesh is complete when they fit.  count32 (int32
    [1]) receives min(nV, V_cap), the vertex count of mesh_normals / netC queries on the device.
    b_min / b_max: None for index space, else the vertices are reconstruction()'s world points
    (v + 0.5) * ((b_max - b_min) / R) + b_min, bit for bit (cubic volumes, R = the side).
    workspace: a McubesWorkspace of the volume's shape (not shared with a run that may still be in flight)."""
    if vol.dim() == 5:
        vol = vol[0, 0]
    _require(vol, torch.float32, None, "vol")
    if vol.dim() != 3:
        raise ValueError("vol must be [D,H,W] or [1,1,D,H,W]; got %s" % (tuple(vol.shape),))
    if not isinstance(workspace, McubesWorkspace) or workspace.shape != tuple(vol.shape) or not workspace.ptr:
        raise ValueError("workspace must be an open McubesWorkspace of shape %s" % (tuple(vol.shape),))
    if verts.dim() != 2 or faces.dim() != 2:
        raise ValueError("verts must be [V_cap,3] and faces [F_cap,3]")
    _require(verts, torch.float32, (verts.shape[0], 3), "verts")
    _require(faces, torch.int32, (faces.shape[0], 3), "faces")
    _require(counts, torch.int64, (2,), "counts")
    _require(count32, torch.int32, (1,), "count32")
    for t in (verts, faces, counts, count32):
        if t.device != vol.device:
            raise ValueError("the volume and the output buffers live on different devices")
    world = None
    if (b_min is None) != (b_max is None):
        raise ValueError("pass both b_min and b_max, or neither")
    if b_min is not None:
        D, H, W = vol.shape
        if not D == H == W:
            raise ValueError("world-space vertices need a cubic volume; got %s" % (tuple(vol.shape),))
        world = (ctypes.c_float * 7)(float(W), *_lib.f3(b_min), *_lib.f3(b_max))
    with _lib.device_guard(vol.device):
        _lib.check(_lib.load().mp_mcubes_run_async(
            workspace.ptr, ctypes.c_void_p(vol.data_ptr()), ctypes.c_float(iso), world, verts.shape[0], faces.shape[0],
            ctypes.c_void_p(verts.data_ptr()), ctypes.c_void_p(faces.data_ptr()), ctypes.c_void_p(counts.data_ptr()),
            ctypes.c_void_p(count32.data_ptr()), _lib.stream_ptr(vol.device)), "mp_mcubes_run_async")


def _check_rounds(rounds, what):
    if isinstance(rounds, bool) or not isinstance(rounds, (int, np.integer)) or rounds < 0:
        raise ValueError("%s must be an integer >= 0; got %r" % (what, rounds))
    return int(rounds)


def _refine_enqueue(net, feat, ws_ptr, vol, iso, b_min, b_max, verts, count32, rounds, calib_tensor, scratch):
    """mp_mesh_refine_async of `rounds` rounds on the current stream (the arguments checked by the callers)"""
    v_cap = verts.shape[0]
    if rounds == 0 or v_cap == 0:
        return
    lib = _lib.load()
    device = vol.device
    need = int(lib.mp_mesh_refine_scratch_bytes(v_cap))
    if scratch is None:
        scratch = torch.empty(need, dtype=torch.uint8, device=device)
    elif scratch.device != device or not scratch.is_contiguous() or scratch.numel() * scratch.element_size() < need:
        raise ValueError("scratch must be a contiguous tensor of at least %d bytes on %s" % (need, device))
    world = (ctypes.c_float * 7)(float(vol.shape[2]), *_lib.f3(b_min), *_lib.f3(b_max))
    with _lib.device_guard(device):
        fh = net.feature_handle(feat)
        _lib.check(lib.mp_mesh_refine_async(
            net.surface_classifier.handle(), fh.ptr, ws_ptr, ctypes.c_void_p(vol.data_ptr()), ctypes.c_float(iso), world,
            ctypes.c_void_p(verts.data_ptr()), ctypes.c_void_p(count32.data_ptr()), v_cap, rounds, _lib.calib12(calib_tensor),
            net._proj(), ctypes.c_float(net.normalizer.scale), net._mode(), ctypes.c_void_p(scratch.data_ptr()),
            _lib.stream_ptr(device)), "mp_mesh_refine_async")


@torch.no_grad()
def refine_mesh_async(net, feat, vol, verts, count32, rounds, b_min, b_max, calib_tensor, iso=0.5, *, workspace, scratch=None):
    """Move the vertices of marching_cubes_async's world-space mesh onto the geometry net's own iso-surface, in place and
    enqueue-only (mp_mesh_refine_async; the algorithm: DESIGN.md §F3.1).  Each vertex stays on its grid edge, which the
    volume's two end values bracket; `rounds` rounds of regula falsi (Illinois) each evaluate the net once per vertex at
    its precision (net.precision, like the volume), starting at the marching-cubes vertex, and the candidate with the
    smallest |sigma - iso| is written back.  Faces and counts are not touched, nor vertices at or beyond min(count32, V_cap).
    rounds = 0 changes nothing, rounds = 1 rewrites the same bits.
    feat: the net's [1,C,H,W] feature map (net.filter(image)[-1][0]); vol, iso, b_min, b_max, verts, count32 and workspace:
    those of the marching_cubes_async call that made the mesh -- the workspace's last run must be that one.
    scratch: None (allocated per call) or a device tensor of at least mp_mesh_refine_scratch_bytes(V_cap) bytes (a CUDA
    graph captures the call with a scratch of its own)."""
    rounds = _check_rounds(rounds, "rounds")
    if vol.dim() == 5:
        vol = vol[0, 0]
    _require(vol, torch.float32, None, "vol")
    if vol.dim() != 3:
        raise ValueError("vol must be [D,H,W] or [1,1,D,H,W]; got %s" % (tuple(vol.shape),))
    if not isinstance(workspace, McubesWorkspace) or workspace.shape != tuple(vol.shape) or not workspace.ptr:
        raise ValueError("workspace must be an open McubesWorkspace of shape %s" % (tuple(vol.shape),))
    D, H, W = vol.shape
    if not D == H == W:
        raise ValueError("world-space vertices need a cubic volume; got %s" % (tuple(vol.shape),))
    if verts.dim() != 2:
        raise ValueError("verts must be [V_cap,3]")
    _require(verts, torch.float32, (verts.shape[0], 3), "verts")
    _require(count32, torch.int32, (1,), "count32")
    for t in (verts, count32, feat):
        if t.device != vol.device:
            raise ValueError("the volume, the mesh buffers and the features live on different devices")
    _refine_enqueue(net, feat, workspace.ptr, vol, iso, b_min, b_max, verts, count32, rounds, calib_tensor, scratch)


@torch.no_grad()
def mesh_normals(net, feats, verts, calib_tensor, precision="auto"):
    """Outward unit normals -grad sigma / |grad sigma| of the geometry net at mesh vertices verts [V,3] (world space, e.g.
    reconstruction()'s), zero where the gradient vanishes -- through mp_mesh_normals_async, the call FrameGraph(mesh_normals=
    True) captures, so both give the same bits.  precision: that of query_gradient ("fp32": the exact kernel, what
    reconstruction(normals=True) uses; "tc" / "auto": the tensor-core program's forward-mode derivative, a frame above the
    head's feature limit differentiated exactly, decided on the device)."""
    from .modeling.MonoPortNet import _MODES
    if precision not in ("fp32", "tc", "auto"):
        raise ValueError("precision must be one of 'fp32', 'tc', 'auto'; got %r" % (precision,))
    feat = feats[-1][0]
    if verts.dim() != 2 or verts.shape[1] != 3:
        raise ValueError("verts must be [V,3]; got %s" % (tuple(verts.shape),))
    if verts.device != feat.device:
        raise ValueError("verts and features live on different devices")
    device = feat.device
    n = verts.shape[0]
    out = torch.empty((n, 3), dtype=torch.float32, device=device)
    if n == 0:
        return out
    v = verts.detach().to(torch.float32).contiguous()
    counts = torch.tensor([n, 0], dtype=torch.int64, device=device)
    count32 = torch.tensor([n], dtype=torch.int32, device=device)
    scratch = torch.empty(3 * n, dtype=torch.float32, device=device)
    with _lib.device_guard(device):
        fh = net.feature_handle(feat)
        _lib.check(_lib.load().mp_mesh_normals_async(
            net.surface_classifier.handle(), fh.ptr, ctypes.c_void_p(v.data_ptr()), ctypes.c_void_p(counts.data_ptr()),
            ctypes.c_void_p(count32.data_ptr()), n, _lib.calib12(calib_tensor), net._proj(), ctypes.c_float(net.normalizer.scale),
            _MODES[precision], ctypes.c_void_p(scratch.data_ptr()), ctypes.c_void_p(out.data_ptr()), _lib.stream_ptr(device)),
            "mp_mesh_normals_async")
    return out


@torch.no_grad()
def mesh_colours(netC, feats_C, verts, calib_tensor):
    """Vertex colours of a mesh, upstream PIFu's gen_mesh_color: netC queried at the vertices verts [V,3] (world space),
    pred * 0.5 + 0.5, as [V,3] -- for mesh_util.save_obj_mesh_with_color / save_ply_mesh(colors=).  FrameGraph(mesh_colours=
    True) computes the same bits inside the captured step."""
    return (netC.query(feats_C, verts.t()[None], calib_tensor)[0][0] * 0.5 + 0.5).t()


def _unit_or_zero(v):
    """rows of v [N,3] scaled to unit length; a zero row stays zero"""
    norm = v.norm(dim=1, keepdim=True)
    return torch.where(norm > 0, v / norm.clamp_min(torch.finfo(v.dtype).tiny), torch.zeros_like(v))


@torch.no_grad()
def reconstruction(net, cuda, calib_tensor, resolution, b_min, b_max, use_octree=False, num_samples=10000,
                   transform=None, feats=None, engine=None, normals=False, refine=0):
    """PIFu-shaped mesh reconstruction (upstream signature, SURVEY.md §8b): evaluate the occupancy field on a
    `resolution`^3 grid over [b_min,b_max] (dense through the fused kernel, or coarse-to-fine when `use_octree`),
    run marching cubes at 0.5, map vertices to world space.  `feats` = net.filter(image) output.
    Returns (verts [V,3] world, faces [F,3], normals, values None) or -1 when the volume is empty
    (upstream returns -1 on marching-cubes failure).  `num_samples` is accepted for signature compatibility
    (the fused kernel needs no batching).
    normals: False -> None.  True -> [V,3] outward unit normals -grad sigma / |grad sigma| at the returned vertices (sigma >
    0.5 is inside), evaluated exactly by the fp32 gradient kernel (MonoPortNet.query_gradient); a vertex where the
    gradient vanishes gets a zero vector.  With `transform` they are mapped like the vertices (inverse transpose of its 3x3
    part, renormalised: a rotation rotates them).
    refine: 0 -> the marching-cubes vertices.  K > 0 -> each vertex moved along its grid edge onto the net's own iso-surface
    by K rounds of refine_mesh_async (DESIGN.md §F3.1) before `normals` and `transform`; faces are unchanged."""
    if feats is None:
        raise ValueError("pass feats=net.filter(image)")
    refine = _check_rounds(refine, "refine")
    R = int(resolution)
    device = torch.device(cuda)
    b_min_t = torch.as_tensor(np.asarray(b_min, dtype=np.float32)).view(3)
    b_max_t = torch.as_tensor(np.asarray(b_max, dtype=np.float32)).view(3)
    if use_octree:
        if engine is None and (R < 3 or (R - 1) & (R - 2)):
            raise ValueError("use_octree=True needs a resolution of 2^k+1 nodes per axis (17, 33, ..., 257, 513: RTL/main.py:187); "
                             "got %d -- use %d, or the dense path (use_octree=False), which takes any resolution"
                             % (R, (1 << max(1, (R - 1).bit_length())) + 1))
        if engine is None:
            from .engine import Seg3dLossless, make_query_func
            res = [R]
            while res[0] > 17 and (res[0] - 1) % 2 == 0:
                res.insert(0, (res[0] - 1) // 2 + 1)
            engine = Seg3dLossless(make_query_func(net), b_min_t.numpy()[None], b_max_t.numpy()[None], res,
                                   balance_value=0.5, faster=False).to(device)
        sdf = engine(im_feat_list=feats, calib_tensor=calib_tensor)
        if sdf is None:
            return -1
        vol = sdf[0, 0]
    else:
        vol = net.query_grid(feats[-1][0], calib_tensor, R, b_min_t, b_max_t)
    if refine and (vol.dtype != torch.float32 or not vol.is_contiguous()):
        vol = vol.float().contiguous()            # (the one copy marching cubes and the refinement both read)
    verts, faces = marching_cubes(vol, 0.5)
    if verts.shape[0] == 0:
        return -1
    # index space -> world:  (v + 0.5)/R * (b_max-b_min) + b_min  (node-centre convention of the engines)
    scale = ((b_max_t - b_min_t) / R).to(verts.device)
    verts = (verts + 0.5) * scale + b_min_t.to(verts.device)
    if refine:
        # on marching_cubes()' per-thread workspace, whose last run read this volume
        count32 = torch.tensor([verts.shape[0]], dtype=torch.int32, device=verts.device)
        _refine_enqueue(net, feats[-1][0], _McubesWorkspace.get(vol.shape, vol.device), vol, 0.5, b_min_t, b_max_t, verts,
                        count32, refine, calib_tensor, None)
    nrm = None
    if normals:
        _, grad = net.query_gradient(feats, verts.t().unsqueeze(0), calib_tensor)
        nrm = _unit_or_zero(-grad[0].t())
    if transform is not None:
        T = torch.as_tensor(transform, dtype=torch.float32, device=verts.device)
        verts = verts @ T[:3, :3].T + T[:3, 3]
        if nrm is not None:
            nrm = _unit_or_zero(nrm @ torch.linalg.inv(T[:3, :3].cpu()).to(nrm.device))      # n' = T^-T n
    return verts, faces, nrm, None


@torch.no_grad()
def make_mat_color(resolution, b_min, b_max, device):
    """Voxel index -> world matrix of the demo (RTL/main.py:201-210): diag((b_max-b_min)/R) with translation b_min."""
    b_min = torch.as_tensor(np.asarray(b_min, dtype=np.float32)).view(3)
    b_max = torch.as_tensor(np.asarray(b_max, dtype=np.float32)).view(3)
    mat = torch.eye(4, dtype=torch.float32)
    length = b_max - b_min
    for a in range(3):
        mat[a, a] = length[a] / resolution
    mat[0:3, 3] = b_min
    return mat.to(device)


@torch.no_grad()
def colorization(netC, feat_tensor_C, X, Y, Z, calib_tensor, norm=None, resolution=257, b_min=(-1, -1, -1),
                 b_max=(1, 1, 1), canvas=None):
    """Direct rendering of the visible surface (RTL/main.py:212-249): either normals as colours, or netC queried at the
    visible vertices (X, Y, R - Z) mapped to world space by mat_color, `pred * 0.5 + 0.5`, scattered into an [R,R,3]
    canvas.  Returns None when there is no surface (X is None), like the reference."""
    if X is None:
        return None
    device = calib_tensor.device
    if canvas is None:
        canvas = torch.ones((resolution, resolution, 3), dtype=torch.float32, device=device)
    image = canvas.clone()
    if norm is not None:
        image[X, Y, :] = ((norm + 1) / 2).clamp(0, 1)
        return image
    head = netC.surface_classifier
    feat = feat_tensor_C[-1][0]
    # the tensor-core program covers maps of at most 65536 texels: a larger map takes the generic route, whose query() runs
    # the exact kernel in "auto" and refuses in "tc"
    if (netC.precision in ("auto", "tc") and not netC.training and X.is_cuda and feat.is_cuda and feat.device == device
            and head.filter_channels[-1] == 3 and head.tc_supported() and feat.shape[-2] * feat.shape[-1] <= 65536):
        # one launch: vertices -> world (mat_color) -> netC -> pred*0.5+0.5 -> canvas  (tensor-core program of the colour head)
        n = int(X.numel())
        rc = _lib.MP_OK
        if n:
            Xc, Yc, Zc = X.contiguous(), Y.contiguous(), Z.float().contiguous()
            with _lib.device_guard(device):
                fh = netC.feature_handle(feat)
                rc = _lib.load().mp_colorize_surface(
                    head.handle(), fh.ptr, ctypes.c_void_p(Xc.data_ptr()), ctypes.c_void_p(Yc.data_ptr()),
                    ctypes.c_void_p(Zc.data_ptr()), n, int(resolution), _lib.f3(b_min), _lib.f3(b_max), _lib.calib12(calib_tensor),
                    netC._proj(), ctypes.c_float(netC.normalizer.scale), ctypes.c_void_p(image.data_ptr()), _lib.stream_ptr(device))
                if rc != _lib.MP_E_RANGE:
                    _lib.check(rc, "mp_colorize_surface")
        if rc != _lib.MP_E_RANGE:
            return image
        # features outside the validated range of the tensor-core colour program: the generic route below (its query()
        # takes the exact fp32 kernel for such a frame)
    samples = _visible_world_points(X, Y, Z, resolution, b_min, b_max, device)
    feats = [[f.to(device) for f in fs] for fs in feat_tensor_C]
    preds = netC.query(feats, points=samples, calibs=calib_tensor)[0]
    image[X, Y, :] = (preds[0] * 0.5 + 0.5).t()
    return image


def _visible_world_points(X, Y, Z, resolution, b_min, b_max, device):
    """forward_vertices("front") output -> the world points [1,3,N] the demo queries there: (X, Y, R - Z) through
    mat_color (RTL/main.py:201-210, 231-233)"""
    from .modeling.geometry import orthogonal
    verts = torch.stack([X.float(), Y.float(), resolution - Z.float()], dim=1)          # RTL/main.py:231-233
    samples = verts.unsqueeze(0).permute(0, 2, 1).contiguous()                          # [1,3,N]
    return orthogonal(samples, make_mat_color(resolution, b_min, b_max, device).unsqueeze(0))


def _surface_normals_device(net, feat, X, Y, Z, calib_tensor, resolution, b_min, b_max, precision):
    """surface_normals in "tc" / "auto": one mp_surface_normals_async call with the vertex count on the device"""
    import ctypes
    from . import _lib
    from .modeling.MonoPortNet import _MODES
    device = calib_tensor.device
    n = X.numel()
    out = torch.empty((n, 3), dtype=torch.float32, device=device)
    if n == 0:
        return out
    Xd, Yd = X.to(device=device, dtype=torch.int64).contiguous(), Y.to(device=device, dtype=torch.int64).contiguous()
    Zd = Z.to(device=device, dtype=torch.float32).contiguous()
    count = torch.tensor([n], dtype=torch.int64, device=device)
    scratch = torch.empty(6 * n + 1, dtype=torch.float32, device=device)
    with _lib.device_guard(device):
        fh = net.feature_handle(feat)
        _lib.check(_lib.load().mp_surface_normals_async(
            net.surface_classifier.handle(), fh.ptr, ctypes.c_void_p(Xd.data_ptr()), ctypes.c_void_p(Yd.data_ptr()),
            ctypes.c_void_p(Zd.data_ptr()), ctypes.c_void_p(count.data_ptr()), n, int(resolution), _lib.f3(b_min),
            _lib.f3(b_max), _lib.calib12(calib_tensor), net._proj(), ctypes.c_float(net.normalizer.scale), _MODES[precision],
            ctypes.c_void_p(scratch.data_ptr()), ctypes.c_void_p(out.data_ptr()), _lib.stream_ptr(device)),
            "mp_surface_normals_async")
    return out


DISPLAY_SIZE = 256          # render_size of the demo's display images (RTL/main.py:257)


class DisplayBuffers:
    """What mp_display_async writes for [R,R,3] canvases on `device`: page-locked host images norm / tex ([S,S,3] float32,
    None for an absent image) and mask ([S,S,1] bool), with their numpy views `arrays`, and the device staging buffer."""

    def __init__(self, has_norm, has_tex, device, size=DISPLAY_SIZE):
        S = self.size = int(size)
        self.norm = torch.empty((S, S, 3), dtype=torch.float32, pin_memory=True) if has_norm else None
        self.tex = torch.empty((S, S, 3), dtype=torch.float32, pin_memory=True) if has_tex else None
        self.mask = torch.empty((S, S, 1), dtype=torch.bool, pin_memory=True)
        self.staging = torch.empty((3 * (int(has_norm) + int(has_tex)) + 1) * S * S, dtype=torch.float32, device=device)
        self.arrays = tuple(None if t is None else t.numpy() for t in (self.norm, self.tex, self.mask))

    def enqueue(self, norm_dev, tex_dev, R, stream):
        """mp_display_async of the canvases (device tensors or None, matching the buffers) on `stream`"""
        def p(t):
            return None if t is None else ctypes.c_void_p(t.data_ptr())
        _lib.check(_lib.load().mp_display_async(p(norm_dev), p(tex_dev), int(R), self.size, p(self.norm), p(self.tex),
                                                p(self.mask), p(self.staging), stream), "mp_display_async")


@torch.no_grad()
def visulization(render_norm, render_tex=None):
    """The demo's display images (RTL/main.py:252-281, the reference's name and return types): each [R,R,3] float32 CUDA
    canvas (either may be None) x255, rotated by torch.rot90(k=1) over dims (0, 1) and resized to 256 x 256 by nearest
    F.interpolate, as numpy float32 [256,256,3]; and mask, numpy bool [256,256,1], False where the three channels of the
    texture image (else the normal image) all equal 255.  (None, None, None) without any image.  One kernel and the
    device-to-host copies of mp_display_async (what FrameGraph(display=True) captures, so both give the same bits) on the
    current stream, then a synchronisation."""
    if render_norm is None and render_tex is None:
        return None, None, None
    imgs = [t for t in (render_norm, render_tex) if t is not None]
    if any(t.device.type != "cuda" for t in imgs):
        raise RuntimeError("monoport_b200.visulization: CUDA tensors only (no CPU path)")
    R = imgs[0].shape[0]
    for t in imgs:
        if t.dtype != torch.float32 or t.dim() != 3 or tuple(t.shape) != (R, R, 3) or t.device != imgs[0].device:
            raise ValueError("visulization takes float32 [R,R,3] canvases of one size on one device; got %s" % (
                [(t.dtype, tuple(t.shape), str(t.device)) for t in imgs],))
    norm = None if render_norm is None else render_norm.detach().contiguous()
    tex = None if render_tex is None else render_tex.detach().contiguous()
    dev = imgs[0].device
    with _lib.device_guard(dev):
        buf = DisplayBuffers(norm is not None, tex is not None, dev)
        buf.enqueue(norm, tex, R, _lib.stream_ptr(dev))
        torch.cuda.current_stream(dev).synchronize()
    return buf.arrays


@torch.no_grad()
def surface_normals(net, feats, X, Y, Z, calib_tensor, resolution=257, b_min=(-1, -1, -1), b_max=(1, 1, 1), precision="fp32"):
    """Exact normals of the visible surface of forward_vertices(sdf, "front"), for colorization(..., norm=...): the
    geometry net's gradient (MonoPortNet.query_gradient) at the points colorization() samples, (X, Y, R - Z) through
    mat_color, returned [N,3] in forward_vertices' frame and sign.  Its normals are -(d/dX, d/dY, d/dZ) of the volume
    in its (X, Y, Z) index axes (finite differences, RTL/recon.py:80-87); Z runs against the world z axis (R - Z above), so
    the normal is -(g_x L_x, g_y L_y, -g_z L_z) / R normalised, with g the world gradient and L = b_max - b_min.  A vertex
    where the gradient vanishes gets a zero vector.  None when there is no surface (X is None).  precision: that of
    query_gradient ("fp32": the exact kernel; "tc" / "auto": the tensor-core program's forward-mode derivative, through
    mp_surface_normals_async -- the launches FrameGraph(render_normals="gradient") captures, so both give the same bits)."""
    if precision not in ("fp32", "tc", "auto"):
        raise ValueError("precision must be one of 'fp32', 'tc', 'auto'; got %r" % (precision,))
    if X is None:
        return None
    device = calib_tensor.device
    if precision != "fp32":
        return _surface_normals_device(net, feats[-1][0].to(device), X, Y, Z, calib_tensor, resolution, b_min, b_max, precision)
    samples = _visible_world_points(X, Y, Z, resolution, b_min, b_max, device)
    feats = [[f.to(device) for f in fs] for fs in feats]
    _, grad = net.query_gradient(feats, samples, calib_tensor, precision=precision)
    length = (torch.as_tensor(np.asarray(b_max, dtype=np.float32)) - torch.as_tensor(np.asarray(b_min, dtype=np.float32)))
    axis = (length.view(3) / resolution * torch.tensor([1.0, 1.0, -1.0])).to(device)
    return _unit_or_zero(-(grad[0].t() * axis))


def view_mats(model_mat, persp_mat, device):
    """ModelMat and PerspMat ([4,4] or [V,4,4] each, numpy or torch; a [4,4] one serves every view) -> the [V,32] float32
    device tensor mp_render_mesh_async reads: each view's ModelMat then PerspMat, row-major (the matrices the reference
    uploads with transpose=GL_TRUE)."""
    mats = []
    for m, what in ((model_mat, "model_mat"), (persp_mat, "persp_mat")):
        t = torch.as_tensor(np.asarray(m.detach().cpu() if torch.is_tensor(m) else m, dtype=np.float32))
        if t.dim() == 2:
            t = t[None]
        if t.dim() != 3 or tuple(t.shape[1:]) != (4, 4) or t.shape[0] < 1:
            raise ValueError("%s must be [4,4] or [V,4,4]; got %s" % (what, tuple(t.shape)))
        mats.append(t)
    M, P = mats
    if M.shape[0] != P.shape[0] and 1 not in (M.shape[0], P.shape[0]):
        raise ValueError("model_mat and persp_mat hold %d and %d views" % (M.shape[0], P.shape[0]))
    V = max(M.shape[0], P.shape[0])
    M, P = M.expand(V, 4, 4), P.expand(V, 4, 4)
    return torch.cat([M.reshape(V, 16), P.reshape(V, 16)], dim=1).contiguous().to(device)


def _view_size(size):
    try:
        W, H = (int(s) for s in size)
    except (TypeError, ValueError):
        raise ValueError("size must be (W, H); got %r" % (size,)) from None
    return W, H


class MeshRenderer:
    """What one mp_render_mesh_async call writes, for meshes of capacity (v_cap, f_cap) drawn from `views` cameras at
    size (W, H): the normal and / or colour images [V,H,W,4] float32 and the scratch.  enqueue() draws the mesh in the
    buffers it is given on the current stream; FrameGraph(views=...) captures it."""

    def __init__(self, f_cap, views, size, has_normals, has_colours, device, clear=(0, 0, 0, 0)):
        W, H = self.size = _view_size(size)
        self.views = int(views)
        lib = _lib.load()
        need = int(lib.mp_render_mesh_scratch_bytes(int(f_cap), self.views, W, H))
        if need < 0:
            raise ValueError("mesh render: bad arguments (f_cap=%d, views=%d, size=%dx%d; sides 1..8192)" % (f_cap, views, W, H))
        self.scratch = torch.empty(need, dtype=torch.uint8, device=device)
        self.normal = torch.empty((self.views, H, W, 4), dtype=torch.float32, device=device) if has_normals else None
        self.colour = torch.empty((self.views, H, W, 4), dtype=torch.float32, device=device) if has_colours else None
        c = [float(x) for x in clear]
        if len(c) != 4:
            raise ValueError("clear must hold 4 values; got %r" % (clear,))
        self.clear = (ctypes.c_float * 4)(*c)

    def enqueue(self, verts, faces, counts, normals, colours, mats, stream):
        def p(t):
            return None if t is None else ctypes.c_void_p(t.data_ptr())
        W, H = self.size
        _lib.check(_lib.load().mp_render_mesh_async(
            p(verts), p(faces), p(counts), verts.shape[0], faces.shape[0], p(normals), p(colours), p(mats), self.views, W, H,
            self.clear, p(self.normal), p(self.colour), p(self.scratch), stream), "mp_render_mesh_async")


@torch.no_grad()
def render_mesh(verts, faces, model_mat, persp_mat, size, normals=None, colours=None, clear=(0, 0, 0, 0)):
    """The mesh (verts [V,3] float32 CUDA, faces [F,3] int32, e.g. reconstruction()'s) drawn from one or more viewer cameras by
    the reference GL renderer's two per-vertex programs (DESIGN.md §F3.2): NormalRender's (n / |n| + 1) / 2 of the
    interpolated (ModelMat [n, 0]).xyz, and ColorRender's interpolated vertex colour, both with alpha 1, GL_LESS depth in
    face order, no culling.  model_mat / persp_mat: [4,4] or [V,4,4] (numpy or torch; a [4,4] one serves every view), the
    numpy matrices the reference passes to its renderer.  size: (W, H).  normals / colours: [V,3] per-vertex attributes
    (either may be None, not both).  clear: the colour of uncovered pixels.
    Returns (normal_img, colour_img): [V,H,W,4] float32 CUDA tensors, row 0 the top of the image (get_color()'s
    orientation), None for an attribute not given.  One mp_render_mesh_async call -- what FrameGraph(views=...) captures,
    so both give the same bits -- with the counts built on the device."""
    if normals is None and colours is None:
        raise ValueError("render_mesh needs normals and / or colours")
    if verts.device.type != "cuda":
        raise RuntimeError("monoport_b200.render_mesh: CUDA tensors only (no CPU path)")
    dev = verts.device
    if verts.dim() != 2 or verts.shape[1] != 3 or faces.dim() != 2 or faces.shape[1] != 3:
        raise ValueError("verts must be [V,3] and faces [F,3]; got %s and %s" % (tuple(verts.shape), tuple(faces.shape)))
    v = verts.detach().to(torch.float32).contiguous()
    f = faces.detach().to(device=dev, dtype=torch.int32).contiguous()
    attrs = []
    for a, what in ((normals, "normals"), (colours, "colours")):
        if a is not None:
            if tuple(a.shape) != tuple(v.shape) or a.device != dev:
                raise ValueError("%s must be [%d,3] on %s; got %s on %s" % (what, v.shape[0], dev, tuple(a.shape), a.device))
            a = a.detach().to(torch.float32).contiguous()
        attrs.append(a)
    mats = view_mats(model_mat, persp_mat, dev)
    counts = torch.tensor([v.shape[0], f.shape[0]], dtype=torch.int64, device=dev)
    with _lib.device_guard(dev):
        r = MeshRenderer(f.shape[0], mats.shape[0], size, normals is not None, colours is not None, dev, clear)
        r.enqueue(v, f, counts, attrs[0], attrs[1], mats, _lib.stream_ptr(dev))
    return r.normal, r.colour
