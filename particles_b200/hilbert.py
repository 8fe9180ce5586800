"""Hilbert sort on the device (particles/hilbert.py).

``hilbert_sort(x)`` restates ``hilbert.hilbert_sort``: for (N,) or (N, 1) points the argsort of x; for (N, d) points,
2 <= d <= 32, each column is standardised by its mean and standard deviation (ddof = 0) and mapped through invlogit,
scaled to integers below floor(2^(62/d)), and the points are sorted by Witham's Hilbert index of those integers
(csrc/smcb_sqmc.cuh), computed in int64 as the reference does: from d = 4 on the index wraps mod 2^64 and the keys
compare as signed values, and that wrapped order is kept.  Points with equal keys come out in any order.
"""
import torch

from . import _lib
from .device import as_device, context, ptr

MAX_DIM = 32


def hilbert_order(xt, keys=False):
    """Order (and, with ``keys`` and d > 1, the unsorted int64 keys) of the component-major (d, N) or (N,) points
    ``xt``, a contiguous float64 CUDA tensor."""
    ctx = context()
    ctx.bind_stream()
    n = xt.shape[-1]
    d = 1 if xt.ndim == 1 else xt.shape[0]
    if not 1 <= d <= MAX_DIM:
        raise NotImplementedError(f"Hilbert keys exist for d = 1..{MAX_DIM} (got d={d})")
    nb = int(ctx.lib.smcb_hilbert_scratch_bytes(n, d))
    if nb < 0:
        raise ValueError(f"hilbert_sort: bad sizes (N={n}, d={d})")
    scratch = torch.empty(nb + 256, dtype=torch.uint8, device=xt.device)
    base = scratch.data_ptr()
    order = torch.empty(n, dtype=torch.int64, device=xt.device)
    k = torch.empty(n, dtype=torch.int64, device=xt.device) if keys and d > 1 else None
    _lib.check(ctx.lib.smcb_hilbert_sort(ctx.handle, ptr(xt), n, d, ptr(order), None if k is None else ptr(k),
                                         base + (-base) % 256))
    return (order, k) if keys else order


def hilbert_sort(x):
    """hilbert.hilbert_sort(x): the (N,) int64 order of the points x, (N,) or (N, d), as a CUDA tensor."""
    x = as_device(x).to(torch.float64)
    xt = x if x.ndim == 1 else x.t()
    if xt.ndim == 2 and xt.shape[0] == 1:
        xt = xt[0]
    return hilbert_order(xt.contiguous())
