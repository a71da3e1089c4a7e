#!/usr/bin/env python
"""Generate tests/golden/display_{257,129,33}.npz: the demo's display images of the UNMODIFIED reference `visulization`
(RTL/main.py:252-281) on seeded canvases, for both images, the normal image only and the texture image only.

RTL/main.py cannot be imported (flask, the streamer and OpenGL at module level), so the function's source is taken out of
it with `ast` and executed on its own with torch, F and np; nothing of it is copied into this repository.  The canvases
hold quantised colours over a background of ones (the texture canvas: ones on the top half, grey below), pixels where only
one or two channels are 1.0, values one ulp either side of 1.0, and NaN pixels.
Run where the reference tree exists:
    python tests/golden/make_display_golden.py
Each file: norm, tex [R,R,3] (the canvases); render_norm, render_tex [256,256,3] and mask_both [256,256,1] of
visulization(norm, tex); mask_norm of visulization(norm, None); mask_tex of visulization(None, tex).  The single-image
calls' images equal render_norm / render_tex (checked here).  Zip entries carry a fixed timestamp, so a rerun
reproduces the files byte for byte.
"""
import ast
import os
import sys
import time
import types
import zipfile

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
sys.path.insert(0, os.path.join(HERE, ".."))

from display_cases import display_canvases  # noqa: E402
from oracle.ref_loader import REF_ROOT  # noqa: E402


def load_visulization():
    path = os.path.join(REF_ROOT, "RTL", "main.py")
    tree = ast.parse(open(path).read(), path)
    fn = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "visulization"]
    assert len(fn) == 1, "visulization not found in %s" % path
    ns = {"torch": torch, "F": F, "np": np}
    exec(compile(ast.Module(body=fn, type_ignores=[]), path, "exec"), ns)
    return ns["visulization"]


class fixed_zip_time:
    """np.savez_compressed stamps each zip entry with the current local time: pin it to 1980-01-01."""

    def __enter__(self):
        self._time = zipfile.time
        zipfile.time = types.SimpleNamespace(time=lambda: 315532800.0, localtime=time.gmtime)
        return self

    def __exit__(self, *exc):
        zipfile.time = self._time
        return False


@torch.no_grad()
def main():
    vis = load_visulization()
    for R, seed in ((257, 1), (129, 2), (33, 3)):
        norm, tex = display_canvases(R, seed)
        rn, rt, mask_both = vis(norm.clone(), tex.clone())
        rn1, none1, mask_norm = vis(norm.clone(), None)
        none2, rt1, mask_tex = vis(None, tex.clone())
        assert none1 is None and none2 is None and vis(None, None) == (None, None, None)
        for a, b in ((rn, rn1), (rt, rt1)):
            assert np.array_equal(a.view(np.int32), b.view(np.int32))
        rec = dict(R=R, norm=norm.numpy(), tex=tex.numpy(), render_norm=np.ascontiguousarray(rn),
                   render_tex=np.ascontiguousarray(rt), mask_both=mask_both, mask_norm=mask_norm, mask_tex=mask_tex)
        out = os.path.join(HERE, "display_%d.npz" % R)
        with fixed_zip_time():
            np.savez_compressed(out, **rec)
        print("display R=%d: %d NaN output values, foreground %d (both) %d (norm) %d (tex) of %d pixels, %d bytes"
              % (R, int(np.isnan(rn).sum() + np.isnan(rt).sum()), mask_both.sum(), mask_norm.sum(), mask_tex.sum(),
                 mask_both.size, os.path.getsize(out)))


if __name__ == "__main__":
    main()
