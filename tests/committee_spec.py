"""Torch restatement of the committee statistics kernels (ab2_committee_moments, ab2_frame_extrema; include/allegro_b200.h)
with the signatures of their wrappers ``_lib.committee_moments`` / ``_lib.frame_extrema``.

``committee_moments`` does the kernel's fp64 operations in the kernel's order (members in member order, starting from
member 0; mu = sum / K; the square-sums divided by K; the g terms added in g order; one rounding at the end).  Each add,
subtract, multiply and divide is one eager torch op on a whole tensor, correctly rounded; the divisions are tensor by
tensor (torch turns a division by a Python scalar into a multiplication by its reciprocal), and the square root is
numpy's (torch's fp64 sqrt on the CPU is not correctly rounded: it misses the last bit for about 0.4 % of inputs).  So
the kernel is held to it bit for bit.  ``frame_extrema`` sums each frame in torch's own order, so its mean matches the
kernel's to rounding only; max and min are exact."""
import numpy as np
import torch

MAX_MEMBERS = 16


def committee_moments(xs, G):
    xs = list(xs)
    K, G = len(xs), int(G)
    if K < 1 or K > MAX_MEMBERS:
        raise RuntimeError(f"committee_moments: {K} members, the kernel takes 1 .. {MAX_MEMBERS}")
    x0 = xs[0]
    x = [t.reshape(-1, G).double() for t in xs]
    kk = torch.full_like(x[0], float(K))
    s = x[0].clone()
    for k in range(1, K):
        s = s + x[k]
    mu = s / kk
    d = x[0] - mu
    q = d * d
    for k in range(1, K):
        d = x[k] - mu
        q = q + d * d
    q = q / kk
    var = q[:, 0].clone()
    for g in range(1, G):
        var = var + q[:, g]
    dev = torch.from_numpy(np.sqrt(var.cpu().numpy())).to(var.device)
    return mu.to(x0.dtype).reshape(x0.shape), dev.to(x0.dtype)


def frame_extrema(x, frame_ptr):
    fp = [int(v) for v in frame_ptr.reshape(-1).tolist()]
    B = len(fp) - 1
    out = torch.zeros(B, 3, dtype=torch.float64, device=x.device)
    xd = x.reshape(-1).double()
    for b in range(B):
        seg = xd[fp[b]:fp[b + 1]]
        if seg.numel():
            out[b, 0], out[b, 1], out[b, 2] = seg.max(), seg.min(), seg.sum() / seg.numel()
    return out.to(x.dtype)
