"""TEST INFRASTRUCTURE ONLY -- torch-CPU restatement of taco_histogram (csrc/summary.cu) with the result layout of
kernels.histogram; the docstring is the specification of the CUDA kernel."""
from __future__ import annotations

import math

import torch


def histogram(res, x, limits):
    """res int64 [nlim + 5]: res[:nlim] = counts of the finite values of x at upper_bound(limits, (double)x), res[nlim] =
    the number of NaN / Inf elements (not binned), res[nlim+1:].view(float64) = {min, max, sum, sum of squares} of the
    widened finite values (DBL_MAX, -DBL_MAX, 0, 0 when there are none).  Sum and sum of squares here are exact (fsum);
    the kernel's are held to a bound against them."""
    nlim = limits.numel()
    xd = x.reshape(-1).double()
    fin = torch.isfinite(xd)
    v = xd[fin]
    idx = torch.searchsorted(limits.double(), v, right=True)
    res[:nlim] = torch.bincount(idx, minlength=nlim)[:nlim]
    res[nlim] = int((~fin).sum())
    dmax = torch.finfo(torch.float64).max
    vn = v.numpy()                               # (squares of widened float32 values are exact in float64)
    stats = torch.tensor([float(v.min()) if len(vn) else dmax, float(v.max()) if len(vn) else -dmax,
                          math.fsum(vn), math.fsum(vn * vn)], dtype=torch.float64)
    res[nlim + 1:] = stats.view(torch.int64)
