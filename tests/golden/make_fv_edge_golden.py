#!/usr/bin/env python
"""Generate tests/golden/fv_{corner,slab,ball01,noise}_{33,65}.npz: forward_vertices of the UNMODIFIED reference
(RTL/recon.py) on volumes that reach the box, in all four directions.

Their surfaces touch the faces, so columns whose first occupied node lies at k < 2 clamp their k - 2 neighbour onto
themselves: v2 == v1 gives Z = 0/0 = NaN and a NaN normal, which the goldens keep.  Same format as make_golden.py's fv_*.npz.
Run where the reference tree exists:
    python tests/golden/make_fv_edge_golden.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))

from oracle import spec  # noqa: E402
from oracle.ref_loader import load_reference  # noqa: E402
from make_golden import checksum  # noqa: E402


@torch.no_grad()
def main():
    ns = load_reference()
    for kind in ("corner", "slab", "ball01", "noise"):
        for R in (33, 65):
            vol = torch.from_numpy(spec.analytic_volume(R, kind))[None, None]
            rec = dict(R=R, kind=kind, vol_checksum=checksum(vol))
            for d in ("front", "back", "left", "right"):
                X, Y, Z, n = ns.forward_vertices(vol.clone(), d)
                Xo, Yo, Zo, no = spec.forward_vertices_ref(vol, d)
                assert torch.equal(X, Xo) and torch.equal(Y, Yo)
                assert torch.equal(Z, Zo) or np.array_equal(Z.numpy(), Zo.numpy(), equal_nan=True)
                assert np.array_equal(n.numpy(), no.numpy(), equal_nan=True)
                rec["X_" + d], rec["Y_" + d], rec["Z_" + d], rec["N_" + d] = X.numpy(), Y.numpy(), Z.numpy(), n.numpy()
                print("forward_vertices %-6s R=%d %-5s -> %5d verts, %4d NaN Z" % (kind, R, d, X.numel(),
                                                                                    int(torch.isnan(Z).sum())))
            np.savez_compressed(os.path.join(HERE, "fv_%s_%d.npz" % (kind, R)), **rec)


if __name__ == "__main__":
    main()
