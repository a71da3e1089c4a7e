"""A numpy restatement of the mesh renderer (monoport_b200/csrc/raster_kernels.cuh; the rules: DESIGN.md §F3.2), operation for
operation in the kernels' order and precision: float32 for the transform, the snapping and the shading, int64 for the edge
functions, float64 for the barycentrics and the depth.  It does not split the faces into the kernels' small and large paths:
both call one coverage-and-depth function, so the fragments of a face do not depend on the path.  render() gives the images
mp_render_mesh_async writes; raster() the depth keys and, for the property tests, the fragment count of every pixel."""
import numpy as np

F = np.float32
GUARD = F(2.0)
MIN_W = F(1.0e-5)
DEPTH_SCALE = 16777215.0
CLEAR_KEY = np.uint64(0xFFFFFFFFFFFFFFFF)


def view_mats(model_mat, persp_mat):
    """[4,4] or [V,4,4] ModelMat and PerspMat (broadcast) -> [V,32] float32, the layout of mats_dev"""
    M = np.asarray(model_mat, dtype=np.float32)
    P = np.asarray(persp_mat, dtype=np.float32)
    M = M[None] if M.ndim == 2 else M
    P = P[None] if P.ndim == 2 else P
    M, P = np.broadcast_arrays(M, P)
    return np.ascontiguousarray(np.concatenate([M.reshape(-1, 16), P.reshape(-1, 16)], axis=1))


def transform(mat, p):
    """clip [N,4] of the points p [N,3]: e = ModelMat [p,1], clip = PerspMat e, rows ((m0 x + m1 y) + m2 z) + m3"""
    M, P = mat[:16].reshape(4, 4), mat[16:].reshape(4, 4)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    e = [((M[i, 0] * x + M[i, 1] * y) + M[i, 2] * z) + M[i, 3] for i in range(4)]
    return np.stack([((P[i, 0] * e[0] + P[i, 1] * e[1]) + P[i, 2] * e[2]) + P[i, 3] * e[3] for i in range(4)], axis=-1)


def snap(ndc, size):
    win = (ndc + F(1)) * (F(size) * F(0.5))
    return np.rint(win * F(256)).astype(np.int64)


def tri_setup(x, y, W, H):
    """x, y int64 [N,3] -> (ok [N], x, y counter-clockwise, bx0, by0, bx1, by1)"""
    area = (x[:, 1] - x[:, 0]) * (y[:, 2] - y[:, 0]) - (y[:, 1] - y[:, 0]) * (x[:, 2] - x[:, 0])
    cw = area < 0
    x, y = x.copy(), y.copy()
    x[cw, 1], x[cw, 2] = x[cw, 2].copy(), x[cw, 1].copy()
    y[cw, 1], y[cw, 2] = y[cw, 2].copy(), y[cw, 1].copy()
    bx0 = np.maximum(-((-(x.min(1) - 128)) >> 8), 0)
    bx1 = np.minimum((x.max(1) - 128) >> 8, W - 1)
    by0 = np.maximum(-((-(y.min(1) - 128)) >> 8), 0)
    by1 = np.minimum((y.max(1) - 128) >> 8, H - 1)
    return (area != 0) & (bx0 <= bx1) & (by0 <= by1), x, y, bx0, by0, bx1, by1


def covered(x, y, i, j):
    """x, y [N,3] counter-clockwise, pixel (i, j) [N] -> bool [N] (edge functions > 0, or = 0 on a top or left edge)"""
    px, py = 256 * i + 128, 256 * j + 128
    ok = np.ones(len(i), dtype=bool)
    for k in range(3):
        a, b = (k + 1) % 3, (k + 2) % 3
        dx, dy = x[:, b] - x[:, a], y[:, b] - y[:, a]
        e = dx * (py - y[:, a]) - dy * (px - x[:, a])
        ok &= (e > 0) | ((e == 0) & ((dy < 0) | ((dy == 0) & (dx < 0))))
    return ok


def barycentrics(c, i, j, W, H):
    """c [N,3,4] float32 clip coordinates of the faces, pixel (i, j) -> b [N,3] float64 (2D-homogeneous form)"""
    px = (2 * i + 1).astype(np.float64) / np.float64(W) - 1.0
    py = (2 * j + 1).astype(np.float64) / np.float64(H) - 1.0
    cd = c.astype(np.float64)
    e = []
    for k in range(3):
        u, v = cd[:, (k + 1) % 3], cd[:, (k + 2) % 3]
        cx = u[:, 1] * v[:, 3] - u[:, 3] * v[:, 1]
        cy = u[:, 3] * v[:, 0] - u[:, 0] * v[:, 3]
        cw = u[:, 0] * v[:, 1] - u[:, 1] * v[:, 0]
        e.append((cx * px + cy * py) + cw)
    s = (e[0] + e[1]) + e[2]
    return np.stack([e[0] / s, e[1] / s, e[2] / s], axis=1)


def lerp3(b, a):
    """((b0 a0 + b1 a1) + b2 a2) in float64; a [N,3(,K)] float32"""
    a = a.astype(np.float64)
    if a.ndim == 3:
        b = b[:, :, None]
    return (b[:, 0] * a[:, 0] + b[:, 1] * a[:, 1]) + b[:, 2] * a[:, 2]


def _plane(v, p):
    x, y, z, w = v
    return [z + w, w - MIN_W, GUARD * w + x, GUARD * w - x, GUARD * w + y, GUARD * w - y][p]


def clip_pieces(c, W, H):
    """the pieces of a face off the direct path: c [3,4] float32 clipped against z >= -w, w >= MIN_W and the guard band
    (Sutherland-Hodgman, each crossing from its inside end), fan-triangulated and snapped -> list of (x [3], y [3])"""
    poly = [tuple(F(q) for q in c[k]) for k in range(3)]
    for p in range(6):
        out = []
        for k in range(len(poly)):
            a, b = poly[k], poly[(k + 1) % len(poly)]
            da, db = _plane(a, p), _plane(b, p)
            ia, ib = bool(da >= 0), bool(db >= 0)
            if ia:
                out.append(a)
            if ia != ib:
                s, e, ds, de = (a, b, da, db) if ia else (b, a, db, da)
                u = ds / (ds - de)
                out.append(tuple(s[q] + u * (e[q] - s[q]) for q in range(4)))
        poly = out
    pieces = []
    for k in range(1, len(poly) - 1):
        vs = (poly[0], poly[k], poly[k + 1])
        pieces.append((np.array([snap(v[0] / v[3], W) for v in vs], dtype=np.int64),
                       np.array([snap(v[1] / v[3], H) for v in vs], dtype=np.int64)))
    return pieces


def _counts(counts, v_cap, f_cap):
    nv, nf = int(counts[0]), int(counts[1])
    return max(0, min(nv, v_cap)), max(0, min(nf, f_cap))


def raster(verts, faces, counts, mats, W, H):
    """-> (keys [V,H,W] uint64 with rows counted from the bottom, fragments [V,H,W] int64: the fragments that passed the
    coverage and depth-range tests at each pixel, large: the number of (view, face) the kernels send down the large path)"""
    verts = np.asarray(verts, dtype=np.float32)
    faces = np.asarray(faces, dtype=np.int32)
    nv, nf = _counts(counts, verts.shape[0], faces.shape[0])
    V = mats.shape[0]
    keys = np.full((V, H * W), CLEAR_KEY, dtype=np.uint64)
    frags = np.zeros((V, H * W), dtype=np.int64)
    large = 0
    idx = faces[:nf].astype(np.int64)
    valid = np.all((idx >= 0) & (idx < nv), axis=1)
    fid = np.nonzero(valid)[0]
    idx = idx[fid]
    with np.errstate(all="ignore"):
        for view in range(V):
            C = transform(mats[view], verts[:nv])
            c = C[idx]                                                     # [F,3,4]
            fin = np.all(np.isfinite(c), axis=(1, 2))
            ndc_x, ndc_y = c[:, :, 0] / c[:, :, 3], c[:, :, 1] / c[:, :, 3]
            direct = fin & np.all((c[:, :, 3] > 0) & (ndc_x >= -GUARD) & (ndc_x <= GUARD) & (ndc_y >= -GUARD)
                                  & (ndc_y <= GUARD), axis=1)
            xs, ys = snap(np.where(direct[:, None], ndc_x, 0), W), snap(np.where(direct[:, None], ndc_y, 0), H)
            ok, x, y, bx0, by0, bx1, by1 = tri_setup(xs, ys, W, H)
            ok &= direct
            small = ok & ((bx1 - bx0 + 1) * (by1 - by0 + 1) <= 16)
            large += int(np.count_nonzero(fin & ~direct)) + int(np.count_nonzero(ok & ~small))
            pieces = [(np.nonzero(ok)[0], x[ok], y[ok], bx0[ok], by0[ok], bx1[ok], by1[ok])]
            for f in np.nonzero(fin & ~direct)[0]:
                for px, py in clip_pieces(c[f], W, H):
                    pok, qx, qy, a0, b0, a1, b1 = tri_setup(px[None], py[None], W, H)
                    if pok[0]:
                        pieces.append((np.array([f]), qx, qy, a0, b0, a1, b1))
            for rows, x_, y_, a0, b0, a1, b1 in pieces:
                bw, bh = a1 - a0 + 1, b1 - b0 + 1
                n = bw * bh
                if n.sum() == 0:
                    continue
                rep = np.repeat(np.arange(len(rows)), n)
                q = np.arange(n.sum()) - np.repeat(np.cumsum(n) - n, n)
                i, j = a0[rep] + q % bw[rep], b0[rep] + q // bw[rep]
                cov = covered(x_[rep], y_[rep], i, j)
                rep, i, j = rep[cov], i[cov], j[cov]
                cf = c[rows[rep]]
                b = barycentrics(cf, i, j, W, H)
                z, w = lerp3(b, cf[:, :, 2]), lerp3(b, cf[:, :, 3])
                zw = (z / w + 1.0) * 0.5
                keep = (zw >= 0.0) & (zw <= 1.0)
                d = np.rint(zw[keep] * DEPTH_SCALE).astype(np.uint64)
                key = (d << np.uint64(32)) | fid[rows[rep[keep]]].astype(np.uint64)
                pix = j[keep] * W + i[keep]
                np.minimum.at(keys[view], pix, key)
                np.add.at(frags[view], pix, 1)
    return keys.reshape(V, H, W), frags.reshape(V, H, W), large


def render(verts, faces, counts, mats, W, H, normals=None, colours=None, clear=(0, 0, 0, 0)):
    """-> (normal [V,H,W,4] or None, colour [V,H,W,4] or None), float32, row 0 the top of the window"""
    verts = np.asarray(verts, dtype=np.float32)
    faces = np.asarray(faces, dtype=np.int32)
    keys, _, _ = raster(verts, faces, counts, mats, W, H)
    V = mats.shape[0]
    clear = np.asarray(clear, dtype=np.float32)
    outs = []
    for is_normal, attr in ((True, normals), (False, colours)):
        if attr is None:
            outs.append(None)
            continue
        attr = np.asarray(attr, dtype=np.float32)
        img = np.empty((V, H, W, 4), dtype=np.float32)
        img[:] = clear
        for view in range(V):
            k = keys[view].reshape(-1)
            pix = np.nonzero(k != CLEAR_KEY)[0]
            j, i = pix // W, pix % W
            idx = faces[(k[pix] & np.uint64(0xFFFFFFFF)).astype(np.int64)].astype(np.int64)
            mat = mats[view]
            c = transform(mat, verts[idx.reshape(-1)]).reshape(-1, 3, 4)
            with np.errstate(all="ignore"):
                b = barycentrics(c, i, j, W, H)
                a = attr[idx]                                                  # [N,3 vertices,3]
                if is_normal:
                    M = mat[:16].reshape(4, 4)
                    a = np.stack([(M[r, 0] * a[..., 0] + M[r, 1] * a[..., 1]) + M[r, 2] * a[..., 2] for r in range(3)], axis=-1)
                    v = lerp3(b, a).astype(np.float32)
                    ln = np.sqrt((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2])
                    rgb = (v / ln[:, None] + F(1)) * F(0.5)
                else:
                    rgb = lerp3(b, a).astype(np.float32)
            img[view, H - 1 - j, i, :3] = rgb
            img[view, H - 1 - j, i, 3] = 1
        outs.append(img)
    return tuple(outs)
