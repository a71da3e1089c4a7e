"""The ordered feature gradient of the training query (MP_VJP_DETERMINISTIC, DESIGN §F1⁗): inputs that crowd the points of an
image into one cell of its map, beside points on the map's last row and column and outside the image, and a restatement of
the documented summation order over a dump of one chunk (the --dump option of tests/emu/emu_fp32.cpp's vjp op)."""
from fractions import Fraction

import numpy as np
import torch

from oracle import spec

# the narrow head of the CPU model's cases (32 channels per map)
NARROW = [33, 64, 48, 1]


def cell_coord(k, f, n):
    """the grid coordinate in [-1, 1] at fraction f of cell k of an axis of n texels (align_corners=True)"""
    return -1.0 + 2.0 * (k + f) / (n - 1)


def one_cell_case(B, N, H, W, chans=NARROW, seed=0, edges=True):
    """B images of N points, calibs=None (the points are (u, v, z) themselves): image b's points lie in cell (3 + b, 5 + 2 b)
    of its H x W map, except -- with `edges` -- the first 8: on the last column, the last row, the far corner and outside.
    -> dict(feats [1][B,C,H,W], points [B,3,N], calib None, Ws, bs, grad_output [1][B,Res,N], last_op, chans, proj)"""
    g = torch.Generator().manual_seed(1000 + seed)
    Ws, bs = spec.make_weights(chans, 1010 + seed)
    feat = torch.cat([spec.make_feat(chans[0] - 1, H, W, 1020 + seed + b) for b in range(B)])
    pts = torch.empty(B, 3, N)
    for b in range(B):
        f = torch.rand(2, N, generator=g, dtype=torch.float64) * 0.9 + 0.05
        pts[b, 0] = cell_coord(5 + 2 * b, f[0], W).float()
        pts[b, 1] = cell_coord(3 + b, f[1], H).float()
        pts[b, 2] = torch.rand(N, generator=g) * 2 - 1
        if edges and N >= 8:
            pts[b, :2, :8] = torch.tensor([[1.0, 0.3, 1.0, 1.5, -0.2, 1.0, -1.0, 0.0],
                                           [-0.1, 1.0, 1.0, 0.0, -1.2, 0.999, 1.0, 1.0]])
    gout = torch.randn(B, chans[-1], N, generator=g)
    return dict(feats=[feat], points=pts, calib=None, Ws=Ws, bs=bs, grad_output=[gout], last_op=spec.LAST_SIGMOID,
                chans=list(chans), proj="orthogonal")


def fma32(w, x, acc):
    """fmaf(w, x, acc) with one rounding: w a float32 scalar, x and acc float32 vectors"""
    w64, x64, a64 = np.float64(w), x.astype(np.float64), acc.astype(np.float64)
    r = w64 * x64 + a64                    # the product is exact in float64, the sum rounded once
    out = r.astype(np.float32)
    # rounding r again to float32 can only differ from one rounding where r lies exactly halfway between two float32s
    o64 = out.astype(np.float64)
    other = np.nextafter(out, np.where(r > o64, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32))
    for i in np.nonzero((r != o64) & (r == (o64 + other.astype(np.float64)) / 2))[0]:
        exact = Fraction(float(w64)) * Fraction(float(x64[i])) + Fraction(float(a64[i]))
        if exact != Fraction(float(r[i])):
            out[i] = max(out[i], other[i]) if exact > Fraction(float(r[i])) else min(out[i], other[i])
    return out


def read_dump(path):
    """a --dump file -> (dX [cols, C], weights [cols, 4], sorted keys [cols], their columns [cols])"""
    raw = open(path, "rb").read()
    cols, C = np.frombuffer(raw[:16], dtype=np.int64)
    o = 16
    dx = np.frombuffer(raw, dtype=np.float32, count=cols * C, offset=o).reshape(cols, C)
    o += 4 * cols * C
    wgt = np.frombuffer(raw, dtype=np.float32, count=cols * 4, offset=o).reshape(cols, 4)
    o += 16 * cols
    keys = np.frombuffer(raw, dtype=np.uint32, count=cols, offset=o)
    order = np.frombuffer(raw, dtype=np.uint32, count=cols, offset=o + 4 * cols)
    assert o + 8 * cols == len(raw)
    return dx, wgt, keys, order


def restate_ordered_dfeat(dx, wgt, keys, order, B, H, W):
    """d features [B,C,H,W] of one chunk in the documented order, from its recorded columns: the sort (a stable sort of the
    columns by key) is checked against numpy's; then texel t = (b, y, x), channel c sums over the cells (y-1, x-1),
    (y-1, x), (y, x-1), (y, x) -- the points' se, sw, ne, nw tap -- and their columns in ascending order s = fmaf(w, dX, s),
    skipping weights of 0, and adds s to the zeroed map when it took a term"""
    cols, C = dx.shape
    key_of = np.empty(cols, dtype=np.uint32)
    key_of[order] = keys
    assert np.array_equal(order, np.argsort(key_of, kind="stable").astype(np.uint32))
    HW = H * W
    members = {}
    for j in range(cols):
        if key_of[j] < B * HW:
            members.setdefault(int(key_of[j]), []).append(j)
    out = np.zeros((B * HW, C), dtype=np.float32)
    for t in range(B * HW):
        y, x = divmod(t % HW, W)
        s, took = np.zeros(C, dtype=np.float32), False
        for cell, ok, tap in ((t - W - 1, y > 0 and x > 0, 3), (t - W, y > 0, 2), (t - 1, x > 0, 1), (t, True, 0)):
            for j in members.get(cell, []) if ok else []:
                if wgt[j, tap] == 0:
                    continue
                s, took = fma32(wgt[j, tap], dx[j], s), True
        if took:
            out[t] = out[t] + s
    return torch.from_numpy(out.reshape(B, H, W, C).transpose(0, 3, 1, 2).copy())


# ---- every radix-pass count of the ordered feature gradient ------------------------------------------------------------------
# a head whose maps have one channel: cheap at every map size
ONE_CHANNEL = [2, 16, 8, 1]


def radix_passes_rule(texels):
    """the passes of the sort over keys up to B * H * W (the key of a point that contributes nothing): 8 bits each, so
    1 + #{k in 1..3 : B * H * W >= 2^(8k)}"""
    return 1 + sum(texels >= 1 << (8 * k) for k in (1, 2, 3))


def spread_case(B, N, H, W, chans=ONE_CHANNEL, seed=0, bands=()):
    """B images of N points, calibs=None: uniform over [-1.1, 1.1]^2 (so some outside the image), the first 8 on the last
    column, the last row, the far corner and outside, the next N // 4 crowded into one cell (the last row of cells in the
    last image, the middle one in the others) and, in the last image, N // 8 more in each band (y0, y1) of texel rows.
    -> the dict of one_cell_case"""
    g = torch.Generator().manual_seed(2000 + seed)
    Ws, bs = spec.make_weights(chans, 2010 + seed)
    feat = torch.cat([spec.make_feat(chans[0] - 1, H, W, 2020 + seed + b) for b in range(B)])
    pts = (torch.rand(B, 3, N, generator=g) * 2.2 - 1.1).contiguous()
    for b in range(B):
        pts[b, :2, :8] = torch.tensor([[1.0, 0.3, 1.0, 1.5, -0.2, 1.0, -1.0, 0.0],
                                       [-0.1, 1.0, 1.0, 0.0, -1.2, 0.999, 1.0, 1.0]])
        k = N // 4
        f = torch.rand(2, k, generator=g, dtype=torch.float64) * 0.9 + 0.05
        pts[b, 0, 8:8 + k] = cell_coord(W // 3, f[0], W).float()
        pts[b, 1, 8:8 + k] = cell_coord(H - 2 if b == B - 1 else H // 2, f[1], H).float()
    o = 8 + N // 4
    for y0, y1 in bands:
        k = N // 8
        y = torch.randint(y0, y1, (k,), generator=g).double()
        f = torch.rand(2, k, generator=g, dtype=torch.float64)
        pts[B - 1, 0, o:o + k] = (f[0] * 2 - 1).float()
        pts[B - 1, 1, o:o + k] = cell_coord(y, f[1], H).clamp(max=1.0).float()
        o += k
    assert o <= N
    gout = torch.randn(B, chans[-1], N, generator=g)
    return dict(feats=[feat], points=pts, calib=None, Ws=Ws, bs=bs, grad_output=[gout], last_op=spec.LAST_SIGMOID,
                chans=list(chans), proj="orthogonal")


# the GPU's batch-against-alone cases: (B, H, W, N, bands of the last image) -> the passes of the batch and of one image.
# B = 3 of 2400 x 2400 reaches keys >= 2^24 in the last image's rows from 2191 on: bands above and below that row.
GPU_RADIX_CASES = {
    "three_vs_two": (2, 200, 200, 3000, ()),
    "four_vs_three": (3, 2400, 2400, 4000, ((2191, 2400), (2100, 2191))),
}


def zero_unit_case(seed=0):
    """the narrow head, calibs=None, where some hidden units have a pre-activation of exactly 0: units 0-7 of layer 0 and
    0-3 of layer 1 have zero weights and bias (0 at every point), units 8-11 of layer 0 see only the depth feature (0 at
    the points with z = 0, a quarter of them).  -> (the dict of one_cell_case, {layer: zero rows})"""
    c = spread_case(2, 400, 16, 20, chans=NARROW, seed=50 + seed)
    Ws, bs = [w.clone() for w in c["Ws"]], [b.clone() for b in c["bs"]]
    Ws[0][:12] = 0.0
    bs[0][:12] = 0.0
    Ws[0][8:12, -1] = torch.tensor([0.7, -0.4, 1.1, -0.9])
    Ws[1][:4] = 0.0
    bs[1][:4] = 0.0
    c["points"][:, 2, ::4] = 0.0
    return dict(c, Ws=Ws, bs=bs), {0: list(range(12)), 1: list(range(4))}
