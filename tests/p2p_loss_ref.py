"""float64 reference of the fused P2P losses (test infrastructure).

Each loss runs the oracle's own elementwise function on float64 inputs (the functions are dtype-generic), so the truth follows the
reference model's formulas rather than a re-derivation; gradients come from float64 autograd.  Scalars the kernels take as fp32
(gamma, alpha, beta, inv_norm) are rounded to fp32 first, so a planted edge such as |diff| == beta is the same edge on both sides.

`fixed_order_sum` restates the kernels' deterministic sum (loss_sum_kernel + block_partial_finish in csrc/ptb_common.cuh) in numpy
fp32.  With terms computed in the kernel's own fp32 operation order (MSE: `mse_terms_f32`) it reproduces the kernel's sum bit for bit,
which pins both the summation order and the grid.
"""
import numpy as np
import torch

from oracle import p2p as op2p, p2p_defaults as odef, p2p_softmax as osm

SUM_BLOCKS, SUM_THREADS = 528, 256          # launch_sum's fixed grid
SUM_GRID = SUM_BLOCKS * SUM_THREADS         # elements per trip of the grid-stride loop
ROWS_PER_TRIP = SUM_BLOCKS * 8              # softmax CE: one warp per row


def f32(v):
    return float(np.float32(v))


def _grad_of(loss, x64):
    loss.backward()
    return loss.detach(), x64.grad


def _row_weighted(l, weight):
    return l if weight is None else l * weight.double()[:, None]


def focal(x, labels, weight, gamma, alpha):
    """sum_m,c sigmoid_focal_loss_elem * weight[m]; a label outside [0, C) is an all-zero row.  -> (sum, d sum / d x) in float64."""
    x64 = x.detach().double().cpu().requires_grad_(True)
    C = x.shape[1]
    lab = labels.cpu().clone()
    lab[(lab < 0) | (lab >= C)] = C                 # the oracle one-hots with C + 1 columns: C is its all-zero row
    l = op2p.sigmoid_focal_loss_elem(x64, lab, f32(gamma), f32(alpha))
    return _grad_of(_row_weighted(l, None if weight is None else weight.cpu()).sum(), x64)


def smooth_l1(pred, target, weight, inv_norm, beta):
    """sum smooth_l1_elem((pred - target) * inv_norm, 0, beta) * weight over (M, 2) points -> (sum, d sum / d pred)."""
    p64 = pred.detach().double().cpu().requires_grad_(True)
    diff = (p64 - target.double().cpu()) * f32(inv_norm)
    l = op2p.smooth_l1_elem(diff, torch.zeros_like(diff), f32(beta))
    if weight is not None:
        l = l * weight.double().cpu()
    return _grad_of(l.sum(), p64)


def mse(pred, target, weight, inv_norm):
    p64 = pred.detach().double().cpu().requires_grad_(True)
    inv = f32(inv_norm)
    l = odef.mse_elem(p64 * inv, target.double().cpu() * inv)
    if weight is not None:
        l = l * weight.double().cpu()
    return _grad_of(l.sum(), p64)


def sigmoid_bce(x, labels, weight, pos_weight=None):
    """sum_m,c binary_cross_entropy_with_logits(x, onehot(labels), pos_weight) * weight[m] -> (sum, d sum / d x)."""
    x64 = x.detach().double().cpu().requires_grad_(True)
    lab = labels.cpu()
    if pos_weight is None:
        l = odef.sigmoid_bce_elem(x64, lab)
    else:
        l = osm.binary_cross_entropy_elem(x64, lab, pos_weight.double().cpu())
    return _grad_of(_row_weighted(l, None if weight is None else weight.cpu()).sum(), x64)


def softmax_ce(x, labels, weight, class_weight=None):
    """sum_m cross_entropy(x[m], labels[m], weight=class_weight) * weight[m] -> (sum, d sum / d x)."""
    x64 = x.detach().double().cpu().requires_grad_(True)
    l = osm.cross_entropy_elem(x64, labels.cpu(), None if class_weight is None else class_weight.double().cpu())
    if weight is not None:
        l = l * weight.double().cpu()
    return _grad_of(l.sum(), x64)


def mse_terms_f32(pred, target, weight, inv_norm):
    """the MSE kernel's terms in its own fp32 order: diff = (pred - target) * inv_norm, term = (diff * diff) * w, one rounding
    per operation (the kernel's __fmul_rn calls cannot be contracted into an FMA)."""
    p = np.asarray(pred, np.float32).ravel()
    t = np.asarray(target, np.float32).ravel()
    diff = (p - t) * np.float32(inv_norm)
    term = diff * diff
    if weight is not None:
        term = term * np.asarray(weight, np.float32).ravel()
    return term


def fixed_order_sum(terms_f32):
    """numpy fp32 restatement of loss_sum_kernel + block_partial_finish over the SUM_BLOCKS x SUM_THREADS grid:
    - element e goes to thread e mod SUM_GRID, which adds its terms in trip order starting from 0;
    - each warp adds with the xor butterfly (16, 8, 4, 2, 1) and lane 0's value is the warp's;
    - thread 0 of a block adds its 8 warp values in order starting from 0;
    - the last block adds the SUM_BLOCKS partials in block order starting from 0, into an output that holds 0."""
    t = np.asarray(terms_f32, np.float32).ravel()
    trips = max(1, -(-t.size // SUM_GRID))
    padded = np.zeros(trips * SUM_GRID, np.float32)
    padded[:t.size] = t
    acc = np.zeros(SUM_GRID, np.float32)
    for k in range(trips):                  # a thread past the end adds nothing; adding +0 leaves a non-zero float as it is
        acc = acc + padded[k * SUM_GRID:(k + 1) * SUM_GRID]
    v = acc.reshape(SUM_BLOCKS, 8, 32)
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[:, :, lanes ^ o]
    warp = v[:, :, 0]
    part = np.zeros(SUM_BLOCKS, np.float32)
    for w in range(8):
        part = part + warp[:, w]
    total = np.float32(0)
    for b in range(SUM_BLOCKS):
        total = np.float32(total + part[b])
    return np.float32(np.float32(0) + total)
