"""Host references of the FCOS kernels (csrc/fcos.cu) for their tests: plain torch / numpy on the CPU.

  * targets          ptb_fcos_targets bit for bit: oracle/fcos.py's target_single per image and level, in chunks of points, laid out in
                     the kernel's row order (level, image, y, x).  Labels int64, targets fp32.
  * norm_sums        ptb_fcos_norm_sums bit for bit: the positive count as an integer and fixed_order_sum of the fp32 centerness terms.
  * box_terms_f32    FcosBoxLoss's per-row term in the kernel's operation order, one rounding per operation in numpy fp32 (linear IoU and
                     GIoU bit for bit; log IoU as float64 -log of the fp32 ic, times w).
  * box_grad64       the float64 analytic gradient of that term times scale and centerness weight, from the kernel's fp32 intermediates
                     (boxes, areas, overlap, union, enclose), with every branch mask taken from the fp32 comparisons the kernel makes, and
                     per component S = sum of |chain-rule products|.
  * ctr_grad_f32     FcosCenternessLoss's gradient bit for bit: fp32(sc * fp32(sigmoid_f32(x) - t)).
  * ctr_terms64      the centerness BCE terms (1 - t) x - log_sigmoid(x) in float64 and the magnitudes of their pieces.
  * decode           ptb_fcos_decode bit for bit: keys, the (key desc, index asc) top-k, the clipped and rescaled boxes, the scores.
"""
import numpy as np
import torch

from oracle import fcos as ofc
from tests.p2p_loss_ref import SUM_BLOCKS, fixed_order_sum, sigmoid_f32

U = 2.0 ** -24
CHUNK_ELEMS = 1 << 22          # point x GT pairs per target_single call
MODES = {'log': 0, 'linear': 1, 'giou': 2}
F32 = np.float32


def _np(t):
    return np.asarray(t.detach().cpu() if torch.is_tensor(t) else t)


# ---------------------------------------------------------------------------------------------------------------------------------
# targets and normalisers
def level_points(sizes, strides):
    """oracle.fcos.points: per level (H*W, 2) fp32, x * stride + stride // 2"""
    return ofc.points(sizes, strides)


def row_points(sizes, strides, B):
    """(N, 2) fp32 point of every row in the kernels' order (level, image, y, x)"""
    return torch.cat([p.repeat(B, 1) for p in level_points(sizes, strides)])


def targets(sizes, strides, gts, gls, ranges, radius, norm_on_bbox, C):
    """ptb_fcos_targets: gts / gls per image ((G, 4) fp32, (G,) int64, G may be 0), ranges (L, 2), radius the centre-sampling radius
    in strides or None -> labels (N,) int64, targets (N, 4) fp32"""
    pts = level_points(sizes, strides)
    rng = torch.as_tensor(np.asarray(ranges, np.float32))
    out_l, out_t = [], []
    for l, p in enumerate(pts):
        cfg = dict(num_classes=C, center_sampling=radius is not None, strides=[strides[l]],
                   center_sample_radius=radius if radius is not None else 1.5)
        for g, gl in zip(gts, gls):
            G = max(int(g.shape[0]), 1)
            step = max(1, CHUNK_ELEMS // G)
            for s in range(0, p.shape[0], step):
                q = p[s:s + step]
                lab, t = ofc.target_single(g, gl, q, rng[l][None].expand(q.shape[0], 2), [q.shape[0]], cfg)
                out_l.append(lab)
                out_t.append(t / strides[l] if norm_on_bbox else t)
    return torch.cat(out_l), torch.cat(out_t)


def _random_gts(g, n, extent, C, lo=2.0, hi=120.0):
    wh = torch.exp(torch.rand(n, 2, generator=g) * float(np.log(hi / lo))) * lo
    c = torch.rand(n, 2, generator=g) * torch.tensor(extent, dtype=torch.float32)
    b = torch.cat([c - wh / 2, c + wh / 2], 1).float()
    return b, torch.randint(0, C, (n,), generator=g)


def _planted_gts(sizes, strides, ranges, C):
    """GTs on the point grid of strides[0] (points x * s + s // 2) and at the ranges' ends, with distinct labels"""
    s = strides[0]
    p = lambda i: float(i * s + s // 2)
    edge = float(ranges[0][1])                                     # the end of range 0 (the start of range 1)
    rows = [
        [p(2), p(2), p(4), p(4)],                                  # edges on grid points: distance 0 is outside
        [p(10) - edge, p(3) - 1.0, p(10) + 1.0, p(3) + 2.0],        # max distance == the end of range 0 and the start of range 1
        [p(14) - edge - 1.0, p(3) - 1.0, p(14) + 1.0, p(3) + 2.0],  # just past it
        [p(20) - 8.0, p(6) - 4.0, p(20) + 8.0, p(6) + 4.0],        # two distinct GTs of equal area over one point: the first wins
        [p(20) - 4.0, p(6) - 8.0, p(20) + 4.0, p(6) + 8.0],
        [p(20) - 2.0, p(6) - 16.0, p(20) + 2.0, p(6) + 16.0],      # a third of the same area
        [10.0, 12.0, 10010.0, 10012.0],                            # area exactly 1e8 == INF: background
        [20.0, 30.0, 20020.0, 6030.0],                             # area 1.2e8 > INF: a positive
        [p(30) - 1.0, p(8) - 1.0, p(30) + 1.0, p(8) + 1.0],        # small against the centre-sampling radius: clipped on all sides
        [p(34) - 0.5, p(8) - 30.0, p(34) + 40.0, p(8) + 0.5],      # long and thin, off-centre
        [-30.0, p(1) - 3.0, p(1) + 2.0, p(1) + 5.0],               # partly outside the map
    ]
    for (h, w), st, (lo, _) in list(zip(sizes, strides, ranges))[1:]:
        qx, qy = float((w - 1) * st + st // 2), float((h - 1) * st + st // 2)
        rows.append([qx - float(lo), qy - 1.0, qx + 1.0, qy + 2.0])  # max distance == the start of the range at the level's last point
    return torch.tensor(rows, dtype=torch.float32), torch.arange(len(rows)) % C


def target_case(kind, seed=0):
    """ptb_fcos_targets inputs: sizes, strides, B, per-image gts / gls (None: no GT in the batch), ranges, radius, norm_on_bbox, C"""
    g = torch.Generator().manual_seed(seed)
    INF = ofc.INF
    if kind == 'one_level':
        sizes, strides, ranges = [(23, 31)], [8], [(-1, INF)]
        B, C, n, radius, norm = 1, 1, [1], None, False
    elif kind == 'odd_strides':
        sizes, strides, ranges = [(40, 52), (24, 31)], [3, 5], [(-1, 16), (16, INF)]
        B, C, n, radius, norm = 3, 511, [20, 0, 33], None, False
    elif kind == 'crowded':
        sizes, strides = [(32, 40), (16, 20), (8, 10), (4, 5), (2, 3)], [4, 8, 16, 32, 64]
        ranges = [(-1, 16), (16, 32), (32, 64), (64, 128), (128, INF)]
        B, C, n, radius, norm = 3, 80, [300, 0, 120], 1.5, False
    elif kind == 'eight_levels':
        sizes = [(40, 44), (24, 26), (10, 11), (16, 18), (8, 9), (6, 6), (4, 5), (2, 3)]
        strides = [3, 5, 12, 8, 16, 24, 32, 64]
        ranges = [(-1, 8), (8, 16), (16, 24), (24, 40), (40, 64), (64, 96), (96, 160), (160, INF)]
        B, C, n, radius, norm = 2, 7, [40, 60], 2.5, True
    elif kind == 'no_gt':
        sizes, strides, ranges = [(16, 20), (8, 10)], [8, 16], [(-1, 32), (32, INF)]
        B, C, n, radius, norm = 2, 3, [0, 0], None, False
    elif kind == 'planted':
        sizes, strides = [(48, 48), (24, 24), (12, 12), (6, 6), (3, 3)], [8, 16, 32, 64, 128]
        ranges = [(-1, 16), (16, 32), (32, 64), (64, 128), (128, INF)]
        B, C, n, radius, norm = 2, 5, [None, None], None, False
    elif kind == 'planted_cs':
        sizes, strides = [(40, 40), (20, 20), (10, 10)], [12, 24, 48]
        ranges = [(-1, 48), (48, 96), (96, INF)]
        B, C, n, radius, norm = 1, 5, [None], 1.5, True
    else:
        raise ValueError(kind)
    extent = (sizes[0][1] * strides[0], sizes[0][0] * strides[0])
    gts, gls = [], []
    for k in n:
        if k is None:
            b, l = _planted_gts(sizes, strides, ranges, C)
        else:
            b, l = _random_gts(g, k, extent, C)
        gts.append(b)
        gls.append(l.long())
    return dict(sizes=sizes, strides=strides, B=B, gts=gts, gls=gls, ranges=ranges, radius=radius, norm=norm, C=C)


def trip_sizes(N, W0=256):
    """two levels of B = 1 with N rows in all: (H0, W0) at stride 8 and (1, rest) at stride 16, rest in [W0, 2 W0)"""
    if N < 2 * W0:
        return [(1, N)], [8]
    h0 = N // W0 - 1
    return [(h0, W0), (1, N - h0 * W0)], [8, 16]


def centerness_f32(t):
    """fcos_centerness in numpy fp32: sqrt(fl(fl(min / max of l, r) * fl(min / max of t, b)))"""
    t = _np(t).astype(F32)
    with np.errstate(invalid='ignore', divide='ignore'):
        lr = np.minimum(t[:, 0], t[:, 2]) / np.maximum(t[:, 0], t[:, 2])
        tb = np.minimum(t[:, 1], t[:, 3]) / np.maximum(t[:, 1], t[:, 3])
        return np.sqrt(lr * tb)


def positive(labels, C):
    lab = _np(labels)
    return (lab >= 0) & (lab < C)


def norm_sums(labels, tgt, C):
    """(the positive count as an int, the fixed-order fp32 sum of the positives' centerness)"""
    pos = positive(labels, C)
    terms = np.where(pos, centerness_f32(tgt), F32(0))
    return int(pos.sum()), fixed_order_sum(terms)


def sum_chain(n):
    """additions on the longest chain of the fixed-order sum of n terms: the thread's trips, the warp butterfly, the block's 8 warps,
    the SUM_BLOCKS partials and the add into the output"""
    trips = max(1, -(-n // (SUM_BLOCKS * 256)))
    return trips + 5 + 8 + SUM_BLOCKS + 1


# ---------------------------------------------------------------------------------------------------------------------------------
# box loss
def _box_f32(points, pred, tgt, mode, overlap_eps, eps):
    """the kernel's fp32 intermediates of every row (numpy fp32, one rounding per operation)"""
    p, d, t = _np(points).astype(F32), _np(pred).astype(F32), _np(tgt).astype(F32)
    px, py = p[:, 0], p[:, 1]
    v = {}
    v['x1'], v['y1'], v['x2'], v['y2'] = px - d[:, 0], py - d[:, 1], px + d[:, 2], py + d[:, 3]
    v['u1'], v['v1'], v['u2'], v['v2'] = px - t[:, 0], py - t[:, 1], px + t[:, 2], py + t[:, 3]
    v['w1'], v['h1'] = v['x2'] - v['x1'], v['y2'] - v['y1']
    v['a1'], v['a2'] = v['w1'] * v['h1'], (v['u2'] - v['u1']) * (v['v2'] - v['v1'])
    ltx, lty = np.maximum(v['x1'], v['u1']), np.maximum(v['y1'], v['v1'])
    rbx, rby = np.minimum(v['x2'], v['u2']), np.minimum(v['y2'], v['v2'])
    v['wx'], v['wy'] = rbx - ltx, rby - lty
    v['iw'], v['ih'] = np.maximum(v['wx'], F32(0)), np.maximum(v['wy'], F32(0))
    v['ov'] = v['iw'] * v['ih']
    v['uni'] = (v['a1'] + v['a2']) - v['ov']
    v['eps_o'] = F32(eps if mode == 'giou' else overlap_eps)
    v['eps'] = F32(eps)
    v['uc'] = np.maximum(v['uni'], v['eps_o'])
    with np.errstate(invalid='ignore', divide='ignore'):
        v['iou'] = v['ov'] / v['uc']
    v['w'] = centerness_f32(t)
    if mode == 'giou':
        v['ex1'], v['ey1'] = np.minimum(v['x1'], v['u1']), np.minimum(v['y1'], v['v1'])
        v['ex2'], v['ey2'] = np.maximum(v['x2'], v['u2']), np.maximum(v['y2'], v['v2'])
        v['ewr'], v['ehr'] = v['ex2'] - v['ex1'], v['ey2'] - v['ey1']
        v['ew'], v['eh'] = np.maximum(v['ewr'], F32(0)), np.maximum(v['ehr'], F32(0))
        v['ea_raw'] = v['ew'] * v['eh']
        v['ea'] = np.maximum(v['ea_raw'], v['eps'])
    return v


def box_terms_f32(points, pred, tgt, labels, C, mode, overlap_eps=1e-6, eps=1e-6):
    """FcosBoxLoss's term of every row: fp32 for 'linear' and 'giou' (bit for bit), float64 -log(ic) * w for 'log'; 0 on negatives"""
    v = _box_f32(points, pred, tgt, mode, overlap_eps, eps)
    pos = positive(labels, C)
    with np.errstate(invalid='ignore', divide='ignore'):
        if mode == 'giou':
            giou = v['iou'] - (v['ea'] - v['uc']) / v['ea']
            term = (F32(1) - giou) * v['w']
        elif mode == 'linear':
            term = (F32(1) - np.maximum(v['iou'], v['eps'])) * v['w']
        else:
            term = -np.log(np.maximum(v['iou'], v['eps']).astype(np.float64)) * v['w'].astype(np.float64)
    return np.where(pos, term, term.dtype.type(0))


def _win(a, b):
    """the gradient share of torch.maximum(a, b) / minimum(b, a) that goes to a: 1, 0.5 on a tie, 0"""
    return np.where(a > b, 1.0, np.where(a == b, 0.5, 0.0))


def box_grad64(points, pred, tgt, labels, C, mode, overlap_eps=1e-6, eps=1e-6, scale=1.0):
    """(grad, S): float64 (N, 4) scale * w * d term / d pred and S (N, 4), the sum of |chain-rule products| of each component.
    The values are the kernel's fp32 intermediates taken as exact; every mask comes from the same fp32 comparison the kernel makes."""
    v = {k: (val.astype(np.float64) if isinstance(val, np.ndarray) else float(val))
         for k, val in _box_f32(points, pred, tgt, mode, overlap_eps, eps).items()}
    f = _box_f32(points, pred, tgt, mode, overlap_eps, eps)
    n = f['x1'].shape[0]
    with np.errstate(invalid='ignore', divide='ignore'):
        uc = v['uc']
        iou = v['ov'] / uc
        zero = np.zeros(n)
        if mode == 'giou':
            g_iou, a_iou = np.full(n, -1.0), np.ones(n)
            g_union = -1.0 / v['ea']
            g_earea = uc / (v['ea'] * v['ea'])
        else:
            keep = f['iou'] >= f['eps']
            if mode == 'linear':
                g_iou = np.where(keep, -1.0, 0.0)
            else:
                g_iou = np.where(keep, -1.0 / iou, 0.0)
            a_iou = np.abs(g_iou)
            g_union = zero
            g_earea = zero
        a_union = np.abs(g_union)
        wu = _win(f['uni'], f['eps_o'])
        g_uni = (g_union + g_iou * (-iou / uc)) * wu
        a_uni = (a_union + a_iou * (iou / uc)) * wu
        g_ov = g_iou / uc - g_uni
        a_ov = a_iou / uc + a_uni
        mx, my = (f['wx'] >= 0).astype(np.float64), (f['wy'] >= 0).astype(np.float64)
        g_iw, g_ih = g_ov * v['ih'] * mx, g_ov * v['iw'] * my
        a_iw, a_ih = a_ov * v['ih'] * mx, a_ov * v['iw'] * my
        h1, w1 = v['h1'], v['w1']
        w_x1, w_x2, w_y1, w_y2 = _win(f['x1'], f['u1']), _win(f['u2'], f['x2']), _win(f['y1'], f['v1']), _win(f['v2'], f['y2'])
        gx1, ax1 = -g_uni * h1 - g_iw * w_x1, a_uni * np.abs(h1) + a_iw * w_x1
        gx2, ax2 = g_uni * h1 + g_iw * w_x2, a_uni * np.abs(h1) + a_iw * w_x2
        gy1, ay1 = -g_uni * w1 - g_ih * w_y1, a_uni * np.abs(w1) + a_ih * w_y1
        gy2, ay2 = g_uni * w1 + g_ih * w_y2, a_uni * np.abs(w1) + a_ih * w_y2
        if mode == 'giou':
            g_ea = g_earea * _win(f['ea_raw'], f['eps'])
            mex, mey = (f['ewr'] >= 0).astype(np.float64), (f['ehr'] >= 0).astype(np.float64)
            g_ew, g_eh = g_ea * v['eh'] * mex, g_ea * v['ew'] * mey
            e_x1, e_x2, e_y1, e_y2 = _win(f['u1'], f['x1']), _win(f['x2'], f['u2']), _win(f['v1'], f['y1']), _win(f['y2'], f['v2'])
            gx1, ax1 = gx1 - g_ew * e_x1, ax1 + g_ew * e_x1
            gx2, ax2 = gx2 + g_ew * e_x2, ax2 + g_ew * e_x2
            gy1, ay1 = gy1 - g_eh * e_y1, ay1 + g_eh * e_y1
            gy2, ay2 = gy2 + g_eh * e_y2, ay2 + g_eh * e_y2
        s = float(np.float32(scale)) * v['w']
        grad = np.stack([-s * gx1, -s * gy1, s * gx2, s * gy2], 1)
        S = np.abs(s)[:, None] * np.stack([ax1, ay1, ax2, ay2], 1)
    pos = positive(labels, C)[:, None]
    return np.where(pos, grad, 0.0), np.where(pos, S, 0.0)


PLANT_EPS = 2.0 ** -20       # the eps the planted rows' ties are built around


def planted_box_rows():
    """(pred, target) (n, 4) fp32 distances (left, top, right, bottom) from the row's point, dyadic so that every box edge, width, area,
    overlap and union is exact in fp32 and float64 while the point stays below 2^12, each planting a tie or clamp edge at eps 2^-20"""
    h, q, e = 2.0 ** -11, 2.0 ** -13, 2.0 ** -12
    rows = [
        ((3, 2.5, 4, 1.5), (3, 2.5, 4, 1.5)),            # pred == target: all four max / min ties, and the enclose ties
        ((4, 1, -2, 1), (2, 2, 2, 2)),                   # touching in x: wx == 0
        ((1, 4, 1, -2), (2, 2, 2, 2)),                   # touching in y: wy == 0
        ((4, 4, -2, -2), (2, 2, 2, 2)),                  # touching on a corner
        ((5, 1, -3, 1), (2, 2, 2, 2)),                   # apart in x: wx < 0
        ((-1, 1, -1, 1), (2, 2, 2, 2)),                  # inverted in x (negative width), overlapping in y
        ((-1, -1, -2, -2), (2, 2, 2, 2)),                # inverted in both
        ((512, 512, 512, 512), (0.5, 0.5, 0.5, 0.5)),    # 1024 x 1024 around 1 x 1: iou == 2^-20
        ((h, h, h, h), (h, h, h, h)),                    # equal 2^-10 squares: union == enclose == 2^-20
        ((q, q, q, q), (e, q, q, e)),                    # union and enclose < 2^-20
        ((0, 0, 0, 0), (2, 1, 3, 4)),                    # ReLU zeros: an empty pred box, iou 0 < eps
        ((0, 2, 3, 0), (1, 2, 1, 2)),                    # zero on two sides
        ((3, 1, 4, 2), (3, 2, 1, 2)),                    # x1 and y2 ties, x2 and y1 wins
        ((1, 2, 1, 2), (3, 3, 3, 3)),                    # pred inside target
        ((5, 6, 7, 8), (1, 1, 1, 1)),                    # target inside pred
        ((2, 0.5, 2, 0.5), (0.5, 2, 0.5, 2)),            # a cross: the enclose is neither box
        ((1, 1, 1, 1), (1, 1, 1, 1)),                    # 2 x 2 squares, equal
        ((4, 4, 4, 4), (2, 2, 2, 2)),                    # nested, one edge each side
    ]
    return (np.array([r[0] for r in rows], np.float32), np.array([r[1] for r in rows], np.float32))


# ---------------------------------------------------------------------------------------------------------------------------------
# centerness loss
def ctr_grad_f32(x, tgt, labels, C, scale=1.0):
    """fp32(sc * fp32(sigmoid_f32(x) - t)) on positive rows, 0 on the others"""
    t = centerness_f32(tgt)
    s = sigmoid_f32(torch.as_tensor(_np(x))).numpy().astype(F32)
    g = F32(scale) * (s - t)
    return np.where(positive(labels, C), g, F32(0))


def ctr_terms64(x, tgt, labels, C):
    """(terms, pieces): float64 (1 - t) x - log_sigmoid(x) on positive rows with t the fp32 centerness target, and the sum of the
    magnitudes of the term's pieces |(1 - t) x|, |min(x, 0)| and log1p(exp(-|x|))"""
    x = _np(x).astype(np.float64)
    t = centerness_f32(tgt).astype(np.float64)
    pos = positive(labels, C)
    a = (1.0 - t) * x
    lp = np.log1p(np.exp(-np.abs(x)))
    terms = a - (np.minimum(x, 0.0) - lp)
    pieces = np.abs(a) + np.abs(np.minimum(x, 0.0)) + lp
    return np.where(pos, terms, 0.0), np.where(pos, pieces, 0.0)


# ---------------------------------------------------------------------------------------------------------------------------------
# decode
def keys_f32(cls, ctr):
    """(B, H, W, C) and (B, H, W, 1) channels-last maps -> (B, H*W) fp32 fl(max_c sigmoid_f32(cls) * sigmoid_f32(ctr))"""
    B, H, W, C = cls.shape
    s = sigmoid_f32(cls.cpu()).reshape(B, H * W, C).max(-1)[0].numpy()
    k = sigmoid_f32(ctr.cpu()).reshape(B, H * W).numpy()
    return s * k


def select(key, k):
    """(B, Q) keys -> (B, k) int64 indices of the top k by (key desc, index asc)"""
    out = []
    for row in key:
        order = np.lexsort((np.arange(row.size), -row))
        out.append(order[:k])
    return np.stack(out)


def decode(cls_maps, reg_maps, ctr_maps, strides, img_hw, nms_pre, scale_factor=None):
    """ptb_fcos_decode: channels-last maps per level -> idx (B, R) int32, boxes (B, R, 4), scores (B, R, C), ctr (B, R), fp32"""
    B, C = cls_maps[0].shape[0], cls_maps[0].shape[3]
    ih = _np(img_hw).astype(F32)
    sf = None if scale_factor is None else _np(scale_factor).astype(F32)
    I, BX, SC, CT = [], [], [], []
    for cls, reg, ctr, st in zip(cls_maps, reg_maps, ctr_maps, strides):
        _, H, W, _ = cls.shape
        Q = H * W
        if 0 < nms_pre < Q:
            idx = select(keys_f32(cls, ctr), nms_pre)
        else:
            idx = np.broadcast_to(np.arange(Q), (B, Q))
        bi = np.arange(B)[:, None]
        sig = sigmoid_f32(cls.cpu()).reshape(B, Q, C).numpy()
        sk = sigmoid_f32(ctr.cpu()).reshape(B, Q).numpy()
        d = reg.cpu().reshape(B, Q, 4).numpy().astype(F32)[bi, idx]
        yi, xi = idx // W, idx % W
        half = F32(int(st) // 2)
        px = xi.astype(F32) * F32(st) + half
        py = yi.astype(F32) * F32(st) + half
        o = np.stack([px - d[..., 0], py - d[..., 1], px + d[..., 2], py + d[..., 3]], -1)
        mx = np.stack([ih[:, 1], ih[:, 0], ih[:, 1], ih[:, 0]], -1)[:, None, :]
        o = np.where(o < 0, F32(0), o)
        o = np.where(o > mx, np.broadcast_to(mx, o.shape), o)
        if sf is not None:
            o = o / sf[:, None, :]
        I.append(idx.astype(np.int32))
        BX.append(o.astype(F32))
        SC.append(sig[bi, idx])
        CT.append(sk[bi, idx])
    return (np.concatenate(I, 1), np.concatenate(BX, 1), np.concatenate(SC, 1), np.concatenate(CT, 1))
