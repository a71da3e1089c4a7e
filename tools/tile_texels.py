"""Distinct bilinear tap texels per 64-point tile of the in-image list of a dense grid query (DESIGN.md §F1, "Nodes outside
the image"), for the shipped brick order and for the z-major order it replaced.  CPU only (numpy):

    python tools/tile_texels.py [--res 257] [--map 128] [--tiles 4000] [--yaw 20 --pitch 33]

Every node of the R^3 grid over [-1, 1]^3 is projected with the camera (u, v = cal[:3, :3] p + cal[:3, 3]); the nodes with
u, v in [-1, 1] are listed in each order, the list is cut into 64-point tiles, and a random sample of tiles counts the
distinct texels of their four taps, (floor(((u + 1) W - 1) / 2) + {0, 1}) per axis, clamped to the map.  Each distinct
texel costs the program one G0 row (1024 fp16) and one map row (256 fp16) of gathers."""
import argparse
import os
import sys

import numpy as np

TILE = 64
BRICK = 4    # the edge of a brick of the in-image list, in nodes (query_tc.cu: kBrick)


def brick_key(ix, iy, iz, R):
    """the position of node (ix, iy, iz) in the brick-major index space of query_tc.cu (BrickSpace), up to a constant:
    x fastest inside a 4x4x4 brick, then the bricks along x, y and z"""
    rb = (R + BRICK - 1) // BRICK
    b = ((iz // BRICK) * rb + iy // BRICK) * rb + ix // BRICK
    return b * BRICK ** 3 + ((iz % BRICK) * BRICK + iy % BRICK) * BRICK + ix % BRICK


def brick_order(nodes, R):
    """node indices (z-major, z slowest) in the order the in-image list holds them"""
    nodes = np.asarray(nodes, dtype=np.int64)
    ix, iy, iz = nodes % R, (nodes // R) % R, nodes // (R * R)
    return nodes[np.argsort(brick_key(ix, iy, iz, R), kind="stable")]


def project(R, cal):
    """u, v of every node of the R^3 grid over [-1, 1]^3, in z-major order (float32, as the node centres of bench.py)"""
    c = ((np.arange(R, dtype=np.float32) / np.float32(R)) + np.float32(1.0 / (2.0 * R))) * np.float32(2.0) - np.float32(1.0)
    z, y, x = np.meshgrid(c, c, c, indexing="ij")
    p = np.stack([x.ravel(), y.ravel(), z.ravel()], 0)
    uv = cal[:2, :3].astype(np.float32) @ p + cal[:2, 3:4].astype(np.float32)
    return uv[0], uv[1]


def texels_per_tile(order, u, v, W, H, tiles, rng):
    """distinct tap texels of `tiles` random full 64-point tiles of the list `order`"""
    n_tiles = len(order) // TILE
    pick = rng.choice(n_tiles, size=min(tiles, n_tiles), replace=False)
    idx = order[: n_tiles * TILE].reshape(n_tiles, TILE)[pick]
    tx = np.floor(((u[idx] + 1.0) * W - 1.0) / 2.0).astype(np.int64)
    ty = np.floor(((v[idx] + 1.0) * H - 1.0) / 2.0).astype(np.int64)
    taps = [np.clip(ty + dy, 0, H - 1) * W + np.clip(tx + dx, 0, W - 1) for dy in (0, 1) for dx in (0, 1)]
    t = np.sort(np.concatenate(taps, 1), 1)
    return 1 + (np.diff(t, axis=1) != 0).sum(1)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--res", type=int, default=257)
    ap.add_argument("--map", type=int, default=128, help="feature map size (square)")
    ap.add_argument("--tiles", type=int, default=4000)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--yaw", type=float, default=None, help="with --pitch: oracle.spec.scene_calib(yaw, pitch); "
                                                           "default: bench.py's camera")
    ap.add_argument("--pitch", type=float, default=None)
    a = ap.parse_args()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    if a.yaw is None:
        import bench
        cal = bench.scene_calib().numpy()[0]
    else:
        from oracle import spec
        cal = spec.scene_calib(a.yaw, a.pitch).numpy()[0]
    R, W = a.res, a.map
    u, v = project(R, cal)
    inside = np.flatnonzero((u >= -1) & (u <= 1) & (v >= -1) & (v <= 1))
    print("R = %d, %d x %d map: %d of %d nodes in the image, %d tiles" % (R, W, W, inside.size, R ** 3, inside.size // TILE))
    for name, order in (("z-major (ascending)", inside), ("4x4x4 bricks (shipped)", brick_order(inside, R))):
        c = texels_per_tile(order, u, v, W, W, a.tiles, np.random.default_rng(a.seed))
        print("  %-24s distinct tap texels per tile: mean %.1f  median %d  p90 %d" %
              (name, c.mean(), int(np.median(c)), int(np.percentile(c, 90))))


if __name__ == "__main__":
    main()
