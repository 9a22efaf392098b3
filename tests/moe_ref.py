"""Plain numpy restatements for the MoE tests: the routing plan, the router's top-k in float64 and the bound on the FP32 logit
error of the route kernel (csrc/moe_kernels.cuh)."""
import numpy as np

U32 = 2.0 ** -24          # unit roundoff of FP32 (round to nearest)


def token_tile(t, e, k):
    mean = -(-t * k // e)
    return 16 if mean <= 16 else (32 if mean <= 32 else 64)


def tiles_max(t, e, k, bn):
    return min(t * k, (t * k + e * (bn - 1)) // bn)


def plan(ids, e, bn, tmax):
    """(dest_row [T,k], tiles [tmax,4]): expert segments in expert order, each padded to a multiple of bn rows, the slots of an
    expert in row-major (token, slot) order -- what torch.where(chosen == e) enumerates."""
    ids = np.asarray(ids)
    flat = ids.reshape(-1)
    dest = np.full(flat.shape, -1, np.int64)
    tiles = np.zeros((tmax, 4), np.int64)
    row, j = 0, 0
    for x in range(e):
        where = np.nonzero(flat == x)[0]
        dest[where] = row + np.arange(len(where))
        for i in range(0, len(where), bn):
            tiles[j] = (x, row + i, min(bn, len(where) - i), 0)
            j += 1
        row += -(-len(where) // bn) * bn
    return dest.reshape(ids.shape), tiles


def logit_error_bound(y, wr):
    """Bound on |fp32 logit - exact logit| of the route kernel for the FP16 row y [H] and router weights wr [E, H].
    Every product of two FP16 values is exact in FP32 (22 significant bits), so only the additions round: lane l of a warp adds
    its H/32 products in sequence with fmaf, then 5 butterfly levels add the lanes -- every term passes through at most
    n = H/32 + 5 rounded additions, and |error| <= gamma_n * sum_j |y_j w_j| with gamma_n = n u / (1 - n u) (Higham, eq. 4.4)."""
    y = np.asarray(y, np.float64)
    wr = np.asarray(wr, np.float64)
    n = y.shape[-1] // 32 + 5
    gamma = n * U32 / (1 - n * U32)
    return gamma * (np.abs(wr) @ np.abs(y))


def topk_f64(logits, k):
    """Top-k of float64 logits (ties to the lower index) and the float64 renormalised softmax weights of the selection."""
    order = np.argsort(-logits, kind="stable")[:k]
    p = np.exp(logits - logits.max())
    sel = p[order]
    return order, sel / sel.sum()
