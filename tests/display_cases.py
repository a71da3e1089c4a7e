"""The demo's display images (visulization, RTL/main.py:252-281) for the tests and tools of FrameGraph(display=True) and
recon.visulization.  TEST INFRASTRUCTURE ONLY.

  visulization_ref  -- a torch restatement, pinned against the reference's own outputs in tests/golden/display_*.npz
                       (generator: tests/golden/make_display_golden.py, run where the reference tree exists);
  display_canvases  -- the seeded [R,R,3] canvases those goldens and the CPU-model tests use.
"""
import numpy as np
import torch
import torch.nn.functional as F


@torch.no_grad()
def visulization_ref(render_norm, render_tex=None, size=256):
    """[R,R,3] canvases (torch, any device; either may be None) -> (norm [size,size,3] float32 numpy or None, tex likewise,
    mask [size,size,1] bool numpy), or three Nones without any image.  Each image is x255, torch.rot90(k=1) over dims
    (0, 1), nearest F.interpolate to size x size; the mask is False where all three channels of the texture image (else
    the normal image) equal 255."""
    if render_norm is None and render_tex is None:
        return None, None, None

    def display(canvas):
        chw = torch.rot90(canvas.detach() * 255.0, 1, [0, 1]).permute(2, 0, 1)
        return F.interpolate(chw[None], size=(size, size))[0].permute(1, 2, 0).cpu().numpy()

    norm = None if render_norm is None else display(render_norm)
    tex = None if render_tex is None else display(render_tex)
    ref = norm if tex is None else tex
    return norm, tex, ~(ref == 255).all(axis=2, keepdims=True)


def display_canvases(R, seed):
    """(norm, tex) [R,R,3] float32: two different silhouettes of quantised colours, with 1.0 in one or two channels of
    some pixels, 1 -/+ 1 ulp in others, and NaN in one or all channels of a few."""
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.arange(R, dtype=torch.float32), torch.arange(R, dtype=torch.float32), indexing="ij")
    c = (R - 1) / 2.0

    def paint(bg, cx, cy, ax, ay):
        img = bg.clone()
        inside = ((xx - cx) / ax) ** 2 + ((yy - cy) / ay) ** 2 <= 1.0
        k = int(inside.sum())
        img[inside] = torch.randint(0, 33, (k, 3), generator=g).float() / 32.0        # 1.0 in some channels by chance
        idx = inside.nonzero()
        pick = idx[torch.randperm(len(idx), generator=g)[:max(8, k // 20)]]
        q = len(pick) // 8
        img[pick[:q, 0], pick[:q, 1], 0] = 1.0                                        # exactly one channel at 1.0
        img[pick[q:2 * q, 0], pick[q:2 * q, 1], :2] = 1.0                             # two channels at 1.0
        img[pick[2 * q:3 * q, 0], pick[2 * q:3 * q, 1], 1:] = 1.0
        img[pick[3 * q:4 * q, 0], pick[3 * q:4 * q, 1]] = float(np.nextafter(np.float32(1), np.float32(0)))
        img[pick[4 * q:5 * q, 0], pick[4 * q:5 * q, 1]] = float(np.nextafter(np.float32(1), np.float32(2)))
        img[pick[5 * q:6 * q, 0], pick[5 * q:6 * q, 1], 2] = float("nan")
        img[pick[6 * q:7 * q, 0], pick[6 * q:7 * q, 1]] = float("nan")
        return img

    ones = torch.ones((R, R, 3))
    norm = paint(ones, c * 0.9, c * 1.1, R * 0.3, R * 0.42)
    half = ones.clone()
    half[R // 2:] = 0.75                                                              # a background that is not ones
    tex = paint(half, c * 1.15, c * 0.95, R * 0.36, R * 0.3)
    return norm, tex
