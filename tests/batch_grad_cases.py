"""The batched point-gradient goldens (tests/golden/bgrad_*.npz: the reference's query() over the B images of a batch_*.npz
case, differentiated by autograd with respect to the points) and the batch case each one extends."""
import os

import numpy as np
import torch

from helpers import GOLDEN
from batch_cases import load_batch_case

BATCH_GRAD_CASES = ["c_rot", "g_mixed", "g_nocalib", "g_persp", "g_rot"]


def load_batch_grad_case(name):
    """load_batch_case(name) and its gradients: value [B,Res,N] (the reference's fp32 query), grad32 / grad64 [B,3,N] (its
    fp32 / fp64 autograd point gradients), grad_output [B,Res,N] | None (ones)"""
    c = load_batch_case(name)
    g = np.load(os.path.join(GOLDEN, "bgrad_%s.npz" % name))
    c.update(value=torch.from_numpy(g["value"]), grad32=torch.from_numpy(g["grad32"]), grad64=torch.from_numpy(g["grad64"]),
             grad_output=torch.from_numpy(g["grad_output"]) if g["grad_output"].size else None)
    return c


def single(case, b):
    """image b of a batched case as a B = 1 case (grad_output [1,Res,N] or None)"""
    c = dict(case, B=1, feat=case["feat"][b:b + 1], points=case["points"][b:b + 1])
    c["calib"] = case["calib"][b:b + 1] if case["calib"] is not None else None
    if case.get("grad_output") is not None:
        c["grad_output"] = case["grad_output"][b:b + 1]
    return c
