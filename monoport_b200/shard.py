"""z-slab sharding of the query grid over GPUs (SURVEY.md §8e): one process per GPU (torch.distributed / NCCL),
every rank evaluates a contiguous range of the z-major node order (a z slab whose boundaries need not fall on plane
boundaries, so the ranks are balanced to within one 128-point tile) with the fused kernel, then ONE all-gather of the
occupancy volume over NVLink -- in place, inside a persistent buffer -- so every rank holds the full [R,R,R] volume for
marching cubes.  No other collective.  `PeerVolumes` / `query_grid_fused` replace even that by peer-memory stores from the
kernel epilogue."""
import torch


def slab_bounds(R, world_size):
    """Contiguous plane ranges [(z0, nz)] -- the first R % world_size ranks get one extra plane (257 = 8*32+1)."""
    base, extra = divmod(int(R), int(world_size))
    out, z = [], 0
    for r in range(world_size):
        nz = base + (1 if r < extra else 0)
        out.append((z, nz))
        z += nz
    return out


def max_slab(R, world_size):
    return -(-int(R) // int(world_size))


def gather_slabs(slab, R, rank, world_size, group=None, out=None):
    """All-gather unequal z slabs into the full [R,R,R] volume.  Slabs are padded to max_slab planes so a single
    `all_gather_into_tensor` moves everything (67.9 MB at 257^3: latency-bound, one collective is the point)."""
    import torch.distributed as dist
    bounds = slab_bounds(R, world_size)
    pad = max_slab(R, world_size)
    dev = slab.device
    send = slab
    if slab.shape[0] != pad:
        send = torch.zeros((pad, R, R), dtype=slab.dtype, device=dev)
        send[:slab.shape[0]] = slab
    recv = torch.empty((world_size * pad, R, R), dtype=slab.dtype, device=dev)
    if world_size == 1:
        recv.copy_(send)
    else:
        dist.all_gather_into_tensor(recv, send.contiguous(), group=group)
    if out is None:
        out = torch.empty((R, R, R), dtype=slab.dtype, device=dev)
    if all(nz == pad for _, nz in bounds):
        out.copy_(recv)
    else:
        for r, (z0, nz) in enumerate(bounds):
            out[z0:z0 + nz] = recv[r * pad:r * pad + nz]
    return out


def range_bounds(R, world_size):
    """Balanced sharding of the R^3 grid: rank r evaluates nodes [r*per, r*per + n_r) of the z-major linear node order,
    per = ceil(R^3 / world) rounded up to a whole number of 128-point tiles.  The ranges are z slabs whose boundaries need
    not fall on plane boundaries (257 = 8*32+1: with whole planes one rank carries 33 planes, the others 32).
    Returns ([(lin0, n)] per rank, per)."""
    total = int(R) ** 3
    per = -(-total // int(world_size))
    per = -(-per // 128) * 128
    out = []
    for r in range(int(world_size)):
        lin0 = min(r * per, total)
        out.append((lin0, max(0, min(per, total - lin0))))
    return out, per


class ShardedVolume:
    """Persistent buffers of the sharded dense grid: ONE flat [world * per] float32 buffer whose first R^3 elements are the
    volume.  `query()` lets the fused kernel write this rank's range straight into its segment of that buffer; `gather()` is
    one in-place all_gather_into_tensor over it -- no padding copies, no reassembly copies, no allocation per frame.
    `.volume` is the [R,R,R] view every rank reads after `gather()`."""

    def __init__(self, R, rank, world_size, device, group=None):
        self.R, self.rank, self.world, self.group = int(R), int(rank), int(world_size), group
        self.bounds, self.per = range_bounds(R, world_size)
        self.flat = torch.empty(self.world * self.per, dtype=torch.float32, device=device)
        self.volume = self.flat[:self.R ** 3].view(self.R, self.R, self.R)
        self.segment = self.flat[self.rank * self.per:(self.rank + 1) * self.per]

    def query(self, net, feat, calibs, b_min, b_max, fh=None):
        lin0, n = self.bounds[self.rank]
        net.query_grid_range(feat, calibs, self.R, b_min, b_max, lin0, n, out=self.segment, fh=fh)
        return self.segment

    def gather(self):
        if self.world > 1:
            import torch.distributed as dist
            dist.all_gather_into_tensor(self.flat, self.segment, group=self.group)     # in place: segment r lives at r*per
        return self.volume


def query_grid_sharded(net, feat, calibs, R, b_min, b_max, rank, world_size, group=None, gather=True, buffers=None):
    """Dense R^3 occupancy volume evaluated range-wise across ranks; returns the full volume (gather=True) or the local
    segment.  Pass a `ShardedVolume` as `buffers` to reuse its memory from frame to frame."""
    sv = buffers if buffers is not None else ShardedVolume(R, rank, world_size, feat.device, group)
    seg = sv.query(net, feat, calibs, b_min, b_max)
    if not gather:
        return seg[:sv.bounds[rank][1]]
    return sv.gather()


# ------------------------------------------------------------------------------------------------------------
# Fused slab exchange (EXPERIMENTAL, opt-in; validated on multi-GPU boxes only): instead of the all-gather every rank's
# kernel stores its slab straight into the full volumes of ALL ranks over NVLink peer memory (mp_query_grid_peers), so
# compute and transfer are one kernel; what is left of the collective is a barrier.
# ------------------------------------------------------------------------------------------------------------
class _DeviceArray:
    """Zero-copy torch view of a raw device pointer (via __cuda_array_interface__)."""

    def __init__(self, ptr, shape):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": "<f4", "data": (int(ptr), False), "version": 2}


class PeerVolumes:
    """`n_sets` (default 2, alternating per frame) full [R,R,R] float32 volumes per rank, each mapped into every other
    rank of the node.  Collective constructor: call it on all ranks of `group` (one process per GPU)."""

    def __init__(self, R, rank, world_size, device, group=None, n_sets=2):
        import ctypes
        import torch.distributed as dist
        from . import _lib
        lib = _lib.load()
        if world_size > 8:
            raise ValueError("at most 8 peers (one NVSwitch node)")
        self.R, self.rank, self.world, self.device, self.group = int(R), rank, world_size, torch.device(device), group
        self._lib, self._own, self._mapped, self.sets, self._frame = lib, [], [], [], 0
        nbytes = self.R ** 3 * 4
        with _lib.device_guard(self.device):
            for _ in range(n_sets):
                ptr = ctypes.c_void_p()
                handle = ctypes.create_string_buffer(64)
                _lib.check(lib.mp_ipc_alloc(nbytes, ctypes.byref(ptr), handle), "mp_ipc_alloc")
                self._own.append(ptr)
                handles = [None] * world_size
                if world_size > 1:
                    dist.all_gather_object(handles, handle.raw, group=group)
                ptrs = []
                for r in range(world_size):
                    if r == rank:
                        ptrs.append(ptr.value)
                        continue
                    p = ctypes.c_void_p()
                    _lib.check(lib.mp_ipc_open(handles[r], ctypes.byref(p)), "mp_ipc_open")
                    self._mapped.append(p)
                    ptrs.append(p.value)
                local = torch.as_tensor(_DeviceArray(ptr.value, (self.R, self.R, self.R)), device=self.device)
                self.sets.append(((ctypes.c_void_p * world_size)(*ptrs), local))
        self._token = torch.zeros(1, dtype=torch.float32, device=self.device)

    def next_set(self):
        s = self.sets[self._frame % len(self.sets)]
        self._frame += 1
        return s

    def barrier(self):
        """Stream-ordered barrier over the ranks: a one-element all-reduce enqueued behind this rank's kernel.  When it
        completes here, every rank's slab kernel has completed, i.e. this rank's volume is fully assembled."""
        if self.world > 1:
            import torch.distributed as dist
            dist.all_reduce(self._token, group=self.group)

    def close(self):
        for p in self._mapped:
            self._lib.mp_ipc_close(p)
        self._mapped = []
        self.sets = []
        for p in self._own:
            self._lib.mp_ipc_free(p)
        self._own = []


def query_grid_fused(net, feat, calibs, R, b_min, b_max, peers, fh=None):
    """Dense R^3 occupancy volume, z-slab sharded over the ranks of `peers` (a PeerVolumes): ONE kernel per rank computes
    its slab and stores it into every rank's volume; returns this rank's full [R,R,R] volume (valid on the current
    stream after the trailing barrier).  Consumers must be ordered on the same stream (the two alternating volume sets
    then make one barrier per frame sufficient)."""
    import ctypes
    from . import _lib
    assert R == peers.R
    lin0, n = range_bounds(R, peers.world)[0][peers.rank]          # balanced ranges of the linear node order
    ptrs, local = peers.next_set()
    with _lib.device_guard(feat.device):
        if fh is None:
            fh = net.feature_handle(feat)
        _lib.check(_lib.load().mp_query_grid_range_peers(
            net.surface_classifier.handle(), fh.ptr, int(R), int(lin0), int(n), _lib.f3(b_min), _lib.f3(b_max),
            _lib.calib12(calibs), net._proj(), ctypes.c_float(net.normalizer.scale), ptrs, peers.world, net._mode(),
            _lib.stream_ptr(feat.device)), "mp_query_grid_range_peers")
    peers.barrier()
    return local
