"""Meshes and cameras of the mesh-render tests (tests/test_mesh_render_cpu.py and _gpu.py): each case is a dict of numpy
arrays -- verts [v_cap,3], faces [f_cap,3] int32, counts (nV, nF), normals / colours [v_cap,3], mats [V,32] (raster_ref
.view_mats), W, H -- that the CPU model, the restatement and mp_render_mesh_async all take as they are."""
import numpy as np

from oracle import spec
from raster_ref import view_mats


def demo_ortho():
    """the demo's orthographic BaseCamera projection (RTL/scene.py:44-50: near 0, far 10, magnification 2)"""
    near, far, scale = 0.0, 10.0, 2.0
    P = np.eye(4)
    P[0, 0] = 2 / scale
    P[1, 1] = 2 / scale
    P[2, 2] = -2 / (far - near)
    P[2, 3] = -(far + near) / (far - near)
    return P


def perspective(fov_deg=90.0, aspect=1.0, near=0.1, far=10.0):
    """an OpenGL perspective projection (gluPerspective's matrix)"""
    f = 1.0 / np.tan(np.radians(fov_deg) / 2)
    P = np.zeros((4, 4))
    P[0, 0] = f / aspect
    P[1, 1] = f
    P[2, 2] = (far + near) / (near - far)
    P[2, 3] = 2 * far * near / (near - far)
    P[3, 2] = -1.0
    return P


def model(pitch_deg=0.0, yaw_deg=0.0, t=(0.0, 0.0, -2.0)):
    """a view matrix: rotation about y (yaw), then about x (pitch), then a translation"""
    a, b = np.radians(pitch_deg), np.radians(yaw_deg)
    Rx = np.array([[1, 0, 0], [0, np.cos(a), -np.sin(a)], [0, np.sin(a), np.cos(a)]])
    Ry = np.array([[np.cos(b), 0, np.sin(b)], [0, 1, 0], [-np.sin(b), 0, np.cos(b)]])
    M = np.eye(4)
    M[:3, :3] = Rx @ Ry
    M[:3, 3] = t
    return M


def golden_mesh(golden_dir, name):
    """marching cubes (the oracle's) of a fv_* golden volume in world space [-1, 1]^3, with the vertex directions from the
    centre as (non-unit) normals and seeded colours"""
    import os
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    R = int(g["R"])
    v, f = spec.marching_cubes_ref(spec.analytic_volume(R, str(g["kind"])), 0.5)
    v = ((v.astype(np.float32) + np.float32(0.5)) * np.float32(2.0 / R) - np.float32(1)).astype(np.float32)
    rng = np.random.default_rng(R)
    return dict(verts=v, faces=f.astype(np.int32), normals=(v - v.mean(0)).astype(np.float32),
                colours=rng.random(v.shape, dtype=np.float32))


def case(mesh, mats, W, H, counts=None):
    out = dict(mesh)
    out.update(mats=np.ascontiguousarray(mats, dtype=np.float32), W=W, H=H,
               counts=np.array(counts if counts is not None else (mesh["verts"].shape[0], mesh["faces"].shape[0]),
                               dtype=np.int64))
    return out


def quad_mesh(half):
    """two triangles of the square [-half, half]^2 at z = 0"""
    v = np.array([[-half, -half, 0], [half, -half, 0], [half, half, 0], [-half, half, 0]], dtype=np.float32)
    f = np.array([[0, 1, 2], [0, 2, 3]], dtype=np.int32)
    return dict(verts=v, faces=f, normals=np.tile(np.float32([[0.2, -0.3, 1.0]]), (4, 1)),
                colours=np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 1, 0]], dtype=np.float32))


def coincident_mesh():
    """one triangle drawn three times at equal depth with different colours and windings: face 0 must win everywhere"""
    v = np.array([[-0.8, -0.8, 0], [0.8, -0.6, 0], [0.1, 0.9, 0]] * 3, dtype=np.float32)
    f = np.array([[3, 4, 5], [0, 2, 1], [6, 7, 8]], dtype=np.int32)
    col = np.repeat(np.eye(3, dtype=np.float32), 3, axis=0)
    return dict(verts=v, faces=f, normals=np.tile(np.float32([[0, 0, 1]]), (9, 1)), colours=col)


def degenerate_mesh():
    """a fan with repeated-index and collinear faces, and vertices with zero normals"""
    rng = np.random.default_rng(3)
    v = rng.uniform(-0.9, 0.9, (12, 3)).astype(np.float32)
    v[9] = v[8] * np.float32(0.5) + v[7] * np.float32(0.5)          # collinear with 7 and 8 in every projection
    f = np.array([[0, 1, 2], [3, 3, 4], [7, 8, 9], [5, 6, 5], [2, 4, 6], [1, 10, 11], [0, 0, 0], [9, 10, 11]], dtype=np.int32)
    n = rng.normal(size=(12, 3)).astype(np.float32)
    n[[1, 10, 11]] = 0
    # and a face in front of the others whose three normals are zero: NaN pixels
    v = np.concatenate([v, np.float32([[-0.5, -0.5, 0.95], [0.5, -0.4, 0.95], [0.0, 0.5, 0.95]])])
    f = np.concatenate([f, np.int32([[12, 13, 14]])])
    n = np.concatenate([n, np.zeros((3, 3), dtype=np.float32)])
    return dict(verts=v, faces=f, normals=n, colours=rng.random((15, 3), dtype=np.float32))


def overflow_mesh(golden_dir):
    """a golden mesh whose counts say fewer vertices and faces than the buffers hold: faces referencing vertices at or
    beyond nV (and a negative index) are skipped, faces at or beyond nF are never read"""
    m = golden_mesh(golden_dir, "fv_sphere_33")
    nv = m["verts"].shape[0] * 2 // 3
    f = m["faces"].copy()
    f[5] = (0, -1, 2)
    return dict(m, faces=f), (nv, f.shape[0] * 3 // 4)


def plane_mesh(n, seed=0):
    """an n x n grid of quads over [-0.9, 0.9]^2 at z = 0, interior vertices jittered, split into triangles along
    alternating diagonals"""
    rng = np.random.default_rng(seed)
    g = np.linspace(-0.9, 0.9, n + 1)
    X, Y = np.meshgrid(g, g, indexing="xy")
    J = rng.uniform(-0.3, 0.3, X.shape + (2,)) * (1.8 / n)
    J[[0, -1], :, :] = 0
    J[:, [0, -1], :] = 0
    v = np.stack([X + J[..., 0], Y + J[..., 1], np.zeros_like(X)], -1).reshape(-1, 3).astype(np.float32)
    faces = []
    for r in range(n):
        for c in range(n):
            a, b, d, e = r * (n + 1) + c, r * (n + 1) + c + 1, (r + 1) * (n + 1) + c, (r + 1) * (n + 1) + c + 1
            faces += [[a, b, e], [a, e, d]] if (r + c) % 2 else [[a, b, d], [b, e, d]]
    return dict(verts=v, faces=np.array(faces, dtype=np.int32), normals=np.tile(np.float32([[0, 0, 1]]), (len(v), 1)),
                colours=np.zeros_like(v))


def cases(golden_dir, size=64):
    """name -> case: the bit-exactness cases of the issue list, at size x size unless stated"""
    O = demo_ortho()
    out = {}
    for name in ("fv_sphere_33", "fv_two_blobs_65", "fv_corner_33", "fv_noise_33"):
        m = golden_mesh(golden_dir, name)
        for pitch in (0, 33):
            out["%s_ortho%d" % (name, pitch)] = case(m, view_mats(model(pitch), O), size, size)
    sphere = golden_mesh(golden_dir, "fv_sphere_33")
    out["persp_near"] = case(sphere, view_mats(model(20, 30, (0.1, 0.0, -0.35)), perspective()), size, size)
    out["quad_large"] = case(quad_mesh(1.5), view_mats(model(0, 0, (0, 0, -2)), O), size, size)
    out["quad_guard"] = case(quad_mesh(3.0), view_mats(model(10, 20, (0, 0, -2)), O), size, size)
    out["quad_persp"] = case(quad_mesh(4.0), view_mats(model(70, 10, (0, -0.2, -0.5)), perspective(60)), size, size)
    out["coincident"] = case(coincident_mesh(), view_mats(model(0, 0, (0, 0, -2)), O), size, size)
    out["degenerate"] = case(degenerate_mesh(), view_mats(model(15, 5), O), size, size)
    m, counts = overflow_mesh(golden_dir)
    out["beyond_count"] = case(m, view_mats(model(33), O), size, size, counts)
    out["views3"] = case(sphere, view_mats(np.stack([model(0), model(33, 45), model(-20, 0, (0.1, 0, -0.6))]),
                                           np.stack([O, O, perspective(70)])), size, size)
    out["nonsquare_96x64"] = case(golden_mesh(golden_dir, "fv_two_blobs_65"),
                                  view_mats(model(33), perspective(60, 96 / 64, 0.5, 5.0)), 96, 64)
    return out
