"""The mesh refinement of DESIGN.md §F3.1 restated in float32 torch ops with the kernels' rounding order
(monoport_b200/csrc/refine_kernels.cuh), over the vertex and edge order of spec.marching_cubes_ref, and a float64 evaluation
of the geometry head for its accuracy figures."""
import numpy as np
import torch

from oracle import spec


def mc_edges(vol, iso=0.5):
    """The edge of every vertex of spec.marching_cubes_ref(vol, iso), in its vertex order: (x, y, z, axis) int64 arrays, the
    owning node and the axis of its +axis edge."""
    vol = np.ascontiguousarray(vol, dtype=np.float32)
    D, H, W = vol.shape
    inside = vol > np.float32(iso)
    act = np.zeros((D, H, W, 3), dtype=bool)
    act[:, :, :-1, 0] = inside[:, :, :-1] != inside[:, :, 1:]
    act[:, :-1, :, 1] = inside[:, :-1, :] != inside[:, 1:, :]
    act[:-1, :, :, 2] = inside[:-1, :, :] != inside[1:, :, :]
    zz, yy, xx, aa = np.nonzero(act)
    return xx, yy, zz, aa


def world_scale(R, b_min, b_max):
    """(scale, b_min) of reconstruction()'s node-centre mapping, as float32 tensors [3]: (b_max - b_min) / R in fp32"""
    lo = torch.tensor(np.asarray(b_min, dtype=np.float32).reshape(3))
    hi = torch.tensor(np.asarray(b_max, dtype=np.float32).reshape(3))
    return (hi - lo) / torch.tensor(np.float32(R)), lo


def edge_world_points(xx, yy, zz, aa, t, scale, lo):
    """world points [V,3] at parameter t [V] along the edges: p = (x, y, z), p[axis] += t, then (p + 0.5) * scale + b_min,
    each step rounded to float32 like the emission"""
    p = torch.stack([torch.as_tensor(xx), torch.as_tensor(yy), torch.as_tensor(zz)], 1).to(torch.float32)
    idx = torch.arange(p.shape[0])
    a = torch.as_tensor(aa, dtype=torch.int64)
    p[idx, a] = p[idx, a] + t
    return (p + 0.5) * scale + lo


@torch.no_grad()
def refine_mesh_ref(query_fn, vol, iso, rounds, b_min, b_max, trace=False):
    """vol [R,R,R] float32 (numpy or tensor) -> (verts [V,3] float32 world, faces [F,3] int32) after `rounds` rounds of the
    refinement, on the CPU.  query_fn(points [3,N] float32) -> [N] values (any device; its float32 values are used).
    trace: also return the candidates' world points of every round, a list of [V,3]."""
    vol = np.ascontiguousarray(vol.cpu().numpy() if torch.is_tensor(vol) else vol, dtype=np.float32)
    R = vol.shape[2]
    _, faces = spec.marching_cubes_ref(vol, iso)
    xx, yy, zz, aa = mc_edges(vol, iso)
    scale, lo = world_scale(R, b_min, b_max)
    iso = torch.tensor(np.float32(iso))
    va = torch.from_numpy(vol[zz, yy, xx])
    vb = torch.from_numpy(vol[zz + (aa == 2), yy + (aa == 1), xx + (aa == 0)])
    t = (iso - va) / (vb - va)
    ta, fa = torch.zeros_like(t), va - iso
    tb, fb = torch.ones_like(t), vb - iso
    tbest, fbest = t.clone(), torch.full_like(t, float("inf"))
    kept = torch.zeros(t.shape, dtype=torch.int64)          # 0 none, 1 the t = 0 side (a), 2 the t = 1 side (b)
    done = torch.zeros(t.shape, dtype=torch.bool)
    pts = edge_world_points(xx, yy, zz, aa, t, scale, lo)
    rows = []
    for r in range(rounds):
        rows.append(pts)
        f = query_fn(pts.t().contiguous()).reshape(-1).to("cpu", torch.float32) - iso
        better = f.abs() < fbest.abs()
        tbest = torch.where(better, t, tbest)
        fbest = torch.where(better, f, fbest)
        if r == rounds - 1:
            break
        done = done | (f == 0)
        side_a = (f > 0) == (fa > 0)
        k = torch.where(side_a, 2, 1)
        ta2, fa2 = torch.where(side_a, t, ta), torch.where(side_a, f, fa)
        tb2, fb2 = torch.where(side_a, tb, t), torch.where(side_a, fb, f)
        twice = kept == k
        fa2 = torch.where(twice & (k == 1), fa2 * 0.5, fa2)
        fb2 = torch.where(twice & (k == 2), fb2 * 0.5, fb2)
        d = fb2 - fa2
        tn = ta2 - (fa2 / d) * (tb2 - ta2)
        tn = torch.where((d == 0) | torch.isnan(tn), (ta2 + tb2) * 0.5, tn)
        lo_t, hi_t = torch.where(ta2 < tb2, ta2, tb2), torch.where(ta2 < tb2, tb2, ta2)
        tn = torch.where(tn < lo_t, lo_t, torch.where(tn > hi_t, hi_t, tn))
        move = ~done
        ta, fa = torch.where(move, ta2, ta), torch.where(move, fa2, fa)
        tb, fb = torch.where(move, tb2, tb), torch.where(move, fb2, fb)
        kept = torch.where(move, k, kept)
        t = torch.where(move, tn, t)
        pts = edge_world_points(xx, yy, zz, aa, t, scale, lo)
    verts = edge_world_points(xx, yy, zz, aa, tbest, scale, lo) if rounds else pts
    return (verts, torch.from_numpy(faces), rows) if trace else (verts, torch.from_numpy(faces))


@torch.no_grad()
def query64(feat, points, calib, Ws, bs, last_op=spec.LAST_SIGMOID, projection="orthogonal", z_scale=spec.Z_SCALE,
            chunk=1 << 16):
    """spec.query_ref in float64 on the inputs' device: feat [1,C,H,W] or [C,H,W], points [3,N] -> [Res,N] float64."""
    feat = (feat[0] if feat.dim() == 4 else feat).double()
    dev = feat.device
    Ws = [w.to(dev, torch.float64) for w in Ws]
    bs = [b.to(dev, torch.float64) for b in bs]
    c = None if calib is None else (calib[0] if calib.dim() == 3 else calib).to(dev, torch.float64)
    out = []
    for s in range(0, points.shape[1], chunk):
        p = points[:, s:s + chunk].to(dev, torch.float64)
        xyz = spec.project_ref(p, c, projection)
        u, v, z = xyz[0], xyz[1], xyz[2]
        in_img = (u >= -1.0) & (u <= 1.0) & (v >= -1.0) & (v <= 1.0)
        x = torch.cat([spec.bilinear_ref(feat, u, v), (z * z_scale)[None]], 0)
        out.append(in_img.double()[None] * spec.mlp_ref(x, Ws, bs, last_op))
    return torch.cat(out, 1)


def edge_roots64(sigma64, vol, iso, b_min, b_max, iters=40):
    """The float64 root of sigma64(points [3,N] float64) - iso on every marching-cubes edge of vol whose float64 end values
    bracket iso, by bisection: -> (mask [V] of such edges, t [V] float64 roots (NaN elsewhere))."""
    vol = np.ascontiguousarray(vol, dtype=np.float32)
    R = vol.shape[2]
    xx, yy, zz, aa = mc_edges(vol, iso)
    lo = torch.tensor(np.asarray(b_min, dtype=np.float64).reshape(3))
    scale = (torch.tensor(np.asarray(b_max, dtype=np.float64).reshape(3)) - lo) / R
    base = torch.stack([torch.as_tensor(xx), torch.as_tensor(yy), torch.as_tensor(zz)], 1).double()
    idx = torch.arange(base.shape[0])
    a = torch.as_tensor(aa, dtype=torch.int64)

    def f_at(t):
        p = base.clone()
        p[idx, a] += t
        return sigma64(((p + 0.5) * scale + lo).t().contiguous()).reshape(-1).cpu() - iso

    t0, t1 = torch.zeros(len(aa), dtype=torch.float64), torch.ones(len(aa), dtype=torch.float64)
    f0, f1 = f_at(t0), f_at(t1)
    mask = (f0 > 0) != (f1 > 0)
    for _ in range(iters):
        tm = 0.5 * (t0 + t1)
        fm = f_at(tm)
        same = (fm > 0) == (f0 > 0)
        t0, f0 = torch.where(same, tm, t0), torch.where(same, fm, f0)
        t1 = torch.where(same, t1, tm)
    return mask, torch.where(mask, 0.5 * (t0 + t1), torch.full_like(t0, float("nan")))


def edge_parameter(verts, vol, iso, b_min, b_max):
    """the parameter t [V] float64 of world vertices verts [V,3] along their marching-cubes edges (the inverse mapping)"""
    vol = np.ascontiguousarray(vol, dtype=np.float32)
    R = vol.shape[2]
    xx, yy, zz, aa = mc_edges(vol, iso)
    lo = torch.tensor(np.asarray(b_min, dtype=np.float64).reshape(3))
    scale = (torch.tensor(np.asarray(b_max, dtype=np.float64).reshape(3)) - lo) / R
    a = torch.as_tensor(aa, dtype=torch.int64)
    p = (verts.cpu().double() - lo) / scale - 0.5
    base = torch.stack([torch.as_tensor(xx), torch.as_tensor(yy), torch.as_tensor(zz)], 1).double()
    return (p - base)[torch.arange(len(aa)), a]
