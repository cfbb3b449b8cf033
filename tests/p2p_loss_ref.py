"""float64 reference of the fused P2P losses (test infrastructure).

Each loss runs the oracle's own elementwise function on float64 inputs (the functions are dtype-generic), so the truth follows the
reference model's formulas rather than a re-derivation; gradients come from float64 autograd.  Scalars the kernels take as fp32
(gamma, alpha, beta, inv_norm) are rounded to fp32 first, so a planted edge such as |diff| == beta is the same edge on both sides.

GHM-C and GHM-R take each element's bin and the per-bin weights as inputs, so the float64 truth weighs every element exactly as the
kernel does; `ghmc_g_f32`, `ghmr_g_f32` and `ghm_bin_step` restate the kernels' fp32 bin decisions, counts, tot, bin weights and
momentum update bit for bit (the bins and weights through oracle/p2p_loss_types.py's own bin_of and bin_weights).

`fixed_order_sum` restates the kernels' deterministic sum (loss_sum_kernel + block_partial_finish in csrc/ptb_common.cuh) in numpy
fp32.  With terms computed in the kernel's own fp32 operation order (MSE: `mse_terms_f32`) it reproduces the kernel's sum bit for bit,
which pins both the summation order and the grid.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import p2p as op2p, p2p_defaults as odef, p2p_loss_types as olt, p2p_softmax as osm

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


def _points_diff(pred, target, row_inv_norm):
    """float64 leaf pred and the normalised difference (pred - target) * fp32(row_inv_norm[m]) of (M, 2) points"""
    p64 = pred.detach().double().cpu().requires_grad_(True)
    inv = torch.as_tensor(np.asarray(row_inv_norm.detach().cpu() if torch.is_tensor(row_inv_norm) else row_inv_norm,
                                     np.float32)).double()
    return p64, (p64 - target.double().cpu()) * inv.reshape(-1, 1)


def _weighted(l, weight):
    return l if weight is None else l * weight.double().cpu()


def l1_rows(pred, target, weight, row_inv_norm):
    """sum l1_elem((pred - target) * row_inv_norm[m]) * weight over (M, 2) points -> (sum, d sum / d pred)."""
    p64, d = _points_diff(pred, target, row_inv_norm)
    return _grad_of(_weighted(olt.l1_elem(d, torch.zeros_like(d)), weight).sum(), p64)


def balanced_l1_rows(pred, target, weight, row_inv_norm, alpha, gamma, beta):
    p64, d = _points_diff(pred, target, row_inv_norm)
    l = olt.balanced_l1_elem(d, torch.zeros_like(d), f32(alpha), f32(gamma), f32(beta))
    return _grad_of(_weighted(l, weight).sum(), p64)


def _elem_weight(bin_idx, bin_weight, valid):
    """each element's GHM weight: its bin's weight, 0 outside every bin and where it is not valid"""
    bi = torch.as_tensor(bin_idx).reshape(-1)
    bw = torch.as_tensor(bin_weight).double().reshape(-1)
    w = torch.where(bi >= 0, bw[bi.clamp(min=0)], torch.zeros((), dtype=torch.float64))
    return torch.where(torch.as_tensor(valid).reshape(-1), w, torch.zeros((), dtype=torch.float64))


def ghmc(x, labels, label_weight, bin_idx, bin_weight):
    """one image's GHMC sum before the division by tot: sum_q,c binary_cross_entropy_with_logits(x, onehot(labels)) * w, w = the
    bin weight of the element's bin (bin_idx (Q * C,), -1: none) where label_weight > 0 -> (sum, d sum / d x) in float64."""
    Q, C = x.shape
    x, labels, label_weight = x.detach().cpu(), labels.cpu(), label_weight.cpu()
    bin_idx = torch.as_tensor(bin_idx).reshape(Q, C)
    rows = max(1, (1 << 23) // C)                # rows per piece: the float64 graph of the 1203-class maps stays a few hundred MB
    total, grad = torch.zeros((), dtype=torch.float64), torch.empty(Q, C, dtype=torch.float64)
    for r in range(0, Q, rows):
        x64 = x[r:r + rows].double().requires_grad_(True)
        t = onehot_f32(labels[r:r + rows], C).double()
        w = _elem_weight(bin_idx[r:r + rows], bin_weight, (label_weight[r:r + rows] > 0)[:, None].expand(-1, C)).reshape(-1, C)
        s, g = _grad_of(F.binary_cross_entropy_with_logits(x64, t, w, reduction='sum'), x64)
        total += s
        grad[r:r + rows] = g
    return total, grad


def ghmr(pred, target, weight, row_inv_norm, mu, bin_idx, bin_weight):
    """one image's GHMR sum before the division by tot: sum (sqrt(d^2 + mu^2) - mu) * w over (Q, 2) points, d = (pred - target) *
    row_inv_norm[q], w = the bin weight of the element's bin where weight > 0 -> (sum, d sum / d pred) in float64."""
    p64, d = _points_diff(pred, target, row_inv_norm)
    m = f32(mu)
    w = _elem_weight(bin_idx, bin_weight, weight.cpu() > 0).reshape(d.shape)
    return _grad_of(((torch.sqrt(d * d + m * m) - m) * w).sum(), p64)


# ---------------------------------------------------------------------------------------------------------------------------------
# exact restatement of the GHM bin step (ghm_hist_kernel + ghm_weights_kernel)
def onehot_f32(labels, C):
    """(..., Q) labels -> (..., Q, C) fp32 one-hot; a label outside [0, C) is an all-zero row"""
    lab = labels.long()
    return ((lab[..., None] == torch.arange(C)) & (lab[..., None] >= 0)).float()


def sigmoid_f32(x):
    """ATen's vectorised CPU sigmoid (0 - x, Sleef expf_u10, 1 + e, division), which the kernels' sigmoidf_acc restates bit for bit,
    on every element.  ATen sends the last elements of each thread's chunk through a scalar loop (std::exp) that rounds differently
    now and then, so this runs on one thread over a length padded to a multiple of 64: no element reaches that loop."""
    flat = x.detach().float().cpu().reshape(-1)
    n = flat.numel()
    pad = torch.zeros((n + 63) // 64 * 64)
    pad[:n] = flat
    nt = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        out = torch.sigmoid(pad)
    finally:
        torch.set_num_threads(nt)
    return out[:n].reshape(x.shape)


def ghmc_g_f32(x, labels):
    """GHMC's g = |sigmoid(x) - t| in CPU fp32 for (..., Q, C) logits: sigmoid_f32 is the kernel's sigmoidf_acc bit for bit and the
    difference and abs are exact fp32 operations."""
    return (sigmoid_f32(x) - onehot_f32(labels.cpu(), x.shape[-1])).abs()


def ghmr_g_f32(pred, target, row_inv_norm, mu):
    """GHMR's g for (..., Q, 2) points in numpy fp32, one rounding per operation as the kernel: d = fp32(fp32(p - t) * inv),
    root = sqrt(fp32(d * d) + fp32(mu * mu)), g = |d / root|.  (mu * mu is the double product rounded once, python's mu ** 2.)"""
    p = np.asarray(pred.detach().cpu() if torch.is_tensor(pred) else pred, np.float32)
    t = np.asarray(target.detach().cpu() if torch.is_tensor(target) else target, np.float32)
    inv = np.asarray(row_inv_norm.detach().cpu() if torch.is_tensor(row_inv_norm) else row_inv_norm, np.float32)
    mu2 = np.float32(float(np.float32(mu)) ** 2)
    with np.errstate(invalid='ignore'):
        d = (p - t) * inv[:, None]
        root = np.sqrt(d * d + mu2)
        return torch.from_numpy(np.abs(d / root))


def bin_index(g, valid, edges):
    """oracle bin_of over a flat g in chunks (the large maps would need an (n, bins) mask at once)"""
    g, valid = g.reshape(-1), valid.reshape(-1)
    chunk = max(1, (1 << 25) // edges.numel())
    out = torch.empty(g.numel(), dtype=torch.long)
    for s in range(0, g.numel(), chunk):
        out[s:s + chunk] = olt.bin_of(g[s:s + chunk], valid[s:s + chunk], edges)
    return out


def ghm_bin_step(g, valid, edges, mmt=0.0, acc_sum=None):
    """ptb_ghm{c,r}_bin_weights restated: g, valid (B, n) -> counts (B, bins + 1) int64 (the last column: valid elements), bin_idx
    (B, n), bin_weight (B, bins) fp32 and tot (B,) fp32; with mmt > 0 acc_sum (bins,) fp32 is updated in place image by image."""
    B = g.shape[0]
    bins = edges.numel() - 1
    counts = torch.zeros(B, bins + 1, dtype=torch.long)
    idx = torch.empty(B, g[0].numel(), dtype=torch.long)
    bw = torch.zeros(B, bins)
    tot = torch.zeros(B)
    for b in range(B):
        idx[b] = bin_index(g[b], valid[b], edges.cpu())
        counts[b, :bins] = torch.bincount(idx[b][idx[b] >= 0], minlength=bins)
        nv = int(valid[b].sum())
        counts[b, bins] = nv
        w, t = olt.bin_weights(counts[b, :bins], nv, mmt, acc_sum)
        bw[b], tot[b] = w, t
    return counts, idx, bw, tot


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
