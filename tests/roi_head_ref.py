"""Host references of the RoI head kernels (csrc/roi_head.cu) for their tests: plain torch / numpy on the CPU.

  * roi_align_fwd     ptb_roi_align_fwd bit for bit: oracle/roi_head.py's roi_align (mmcv's fp32 CPU arithmetic, pinned to
                      torchvision) on each level, plus the kernel's two extensions: a RoI whose batch index (truncated toward zero) lies
                      outside [0, B) has zero features, and with L > 1 a RoI whose scale is NaN has level -1 and zero features.
  * roi_align_bwd64   the exact gradient of the kernel's own sample weights: the same roi_align on float64 maps under autograd (the
                      positions and weights stay fp32, the accumulation is float64), S_e = sum |terms| of every map element from a
                      second pass with |grad_y|, and the number of non-zero terms each element receives (term_counts).
  * bbox2delta_f32    box_coder.cuh's bbox2delta in its fp32 operation order (log correctly rounded).
  * argmax_rule       the accuracy's prediction: torch.argmax on the CPU (first NaN, else first maximum).
  * decode64          ptb_roi_decode in float64 from the fp32 inputs.
  * bbox_loss64       RoIBoxLoss (loss_terms.cuh) in float64: the sum and its gradient.
The RoIAlign passes run in chunks of RoIs: the oracle's tap gather is (n, C, out, gh, out, gw) and its map gather (n, C, H, W)."""
import numpy as np
import torch

from oracle import roi_head as orh

U = 2.0 ** -24
CHUNK_ELEMS = 1 << 22          # floats per RoIAlign chunk (gathered maps plus sample taps)


def levels(rois, L, finest_scale):
    """the kernel's level of each RoI (int64): 0 when L == 1, else map_roi_levels with -1 where the scale is NaN"""
    if L == 1:
        return torch.zeros(rois.shape[0], dtype=torch.int64)
    s = torch.sqrt((rois[:, 3] - rois[:, 1]) * (rois[:, 4] - rois[:, 2]))
    lv = orh.map_roi_levels(rois, L, finest_scale)
    return torch.where(torch.isnan(s), torch.full_like(lv, -1), lv)


def _grid(rois, out, sc, sampling_ratio):
    """(gh, gw) of each RoI, as roi_geom forms them"""
    sc = torch.tensor(sc, dtype=torch.float32)
    sw, sh = rois[:, 1] * sc - 0.5, rois[:, 2] * sc - 0.5
    bw, bh = ((rois[:, 3] * sc - 0.5) - sw) / out, ((rois[:, 4] * sc - 0.5) - sh) / out
    if sampling_ratio > 0:
        n = torch.full((rois.shape[0],), sampling_ratio, dtype=torch.int64)
        return n, n
    return torch.ceil(bh).long(), torch.ceil(bw).long()


def _chunks(idx, rois, out, sc, sampling_ratio, per_roi):
    """split the RoI indices idx into runs whose gathers stay near CHUNK_ELEMS floats"""
    if idx.numel() == 0:
        return []
    gh, gw = _grid(rois[idx], out, sc, sampling_ratio)
    cost = (per_roi[0] + per_roi[1] * (gh.clamp(min=0) * gw.clamp(min=0)).clamp(min=1)).tolist()
    runs, start, acc = [], 0, 0
    for i, c in enumerate(cost):
        if i > start and acc + c > CHUNK_ELEMS:
            runs.append(idx[start:i])
            start, acc = i, 0
        acc += c
    runs.append(idx[start:])
    return runs


def _live(rois, B, lv):
    b = rois[:, 0].long()
    return (lv >= 0) & (b >= 0) & (b < B)


def roi_align_fwd(maps_nhwc, strides, rois, out, sampling_ratio, finest_scale):
    """ptb_roi_align_fwd: maps_nhwc per level (B, H, W, C) fp32 -> features (R, C, out, out) fp32, levels (R,) int64"""
    maps = [m.cpu().permute(0, 3, 1, 2) for m in maps_nhwc]
    rois = rois.cpu()
    L, B, C = len(maps), maps[0].shape[0], maps[0].shape[1]
    lv = levels(rois, L, finest_scale)
    live = _live(rois, B, lv)
    y = torch.zeros((rois.shape[0], C, out, out), dtype=torch.float32)
    for l in range(L):
        idx = (live & (lv == l)).nonzero().squeeze(1)
        H, W = maps[l].shape[2:]
        sc = 1.0 / strides[l]
        for run in _chunks(idx, rois, out, sc, sampling_ratio, (C * H * W, 8 * C * out * out)):
            y[run] = orh.roi_align(maps[l], rois[run], out, sc, sampling_ratio)
    return y, lv


def term_counts(map_shapes, strides, rois, lv, out, sampling_ratio):
    """per level (B, H, W) int64: how many non-zero terms (RoI, bin, sample, tap) the backward adds into each map element (of every
    channel).  Sample positions, the outside test, the clamps and the weights as roi_align forms them."""
    counts = []
    B = map_shapes[0][0]
    live = _live(rois, B, lv)
    for l, (_, H, W, _) in enumerate(map_shapes):
        cnt = torch.zeros(B * H * W, dtype=torch.int64)
        idx = (live & (lv == l)).nonzero().squeeze(1)
        sc = torch.tensor(1.0 / strides[l], dtype=torch.float32)
        r = rois[idx]
        gh, gw = _grid(r, out, 1.0 / strides[l], sampling_ratio)
        sw, sh = r[:, 1] * sc - 0.5, r[:, 2] * sc - 0.5
        bw, bh = ((r[:, 3] * sc - 0.5) - sw) / out, ((r[:, 4] * sc - 0.5) - sh) / out
        p = torch.arange(out, dtype=torch.float32)
        for g_h, g_w in sorted(set(zip(gh.tolist(), gw.tolist()))):
            if g_h <= 0 or g_w <= 0:
                continue
            k = ((gh == g_h) & (gw == g_w)).nonzero().squeeze(1)

            def axis(start, bin_, g, size):
                v = (start[k, None] + p[None, :] * bin_[k, None])[:, :, None] + \
                    ((torch.arange(g, dtype=torch.float32) + 0.5)[None, :] * bin_[k, None] / float(g))[:, None, :]   # (n, out, g)
                ok = ~((v < -1.0) | (v > size))
                v = torch.where(v <= 0, torch.zeros_like(v), v)
                lo = v.long()
                top = lo >= size - 1
                lo = torch.where(top, torch.full_like(lo, size - 1), lo)
                hi = torch.where(top, lo, lo + 1)
                v = torch.where(top, lo.float(), v)
                frac = v - lo.float()
                return ok.flatten(1), lo.flatten(1), hi.flatten(1), frac.flatten(1), (1.0 - frac).flatten(1)
            oy, yl, yh, ly, hy = axis(sh, bh, g_h, H)
            ox, xl, xh, lx, hx = axis(sw, bw, g_w, W)
            base = r[k, 0].long()[:, None, None] * (H * W)
            ok = oy[:, :, None] & ox[:, None, :]
            for yi, wy in ((yl, hy), (yh, ly)):
                for xi, wx in ((xl, hx), (xh, lx)):
                    w = wy[:, :, None] * wx[:, None, :]
                    flat = base + yi[:, :, None] * W + xi[:, None, :]
                    cnt += torch.bincount(flat[ok & (w != 0)], minlength=B * H * W)
        counts.append(cnt.view(B, H, W))
    return counts


def roi_align_bwd64(map_shapes, strides, rois, lv, out, sampling_ratio, grad_y):
    """ptb_roi_align_bwd in float64 on the kernel's own weights: per level (grad (B, H, W, C), S (B, H, W, C), counts (B, H, W)) with
    S = sum |grad_y * w / count| over the terms of each element"""
    rois, grad_y = rois.cpu(), grad_y.cpu().double()
    B = map_shapes[0][0]
    live = _live(rois, B, lv)
    counts = term_counts(map_shapes, strides, rois, lv, out, sampling_ratio)
    res = []
    for l, (_, H, W, C) in enumerate(map_shapes):
        f = torch.zeros((B, C, H, W), dtype=torch.float64, requires_grad=True)
        g, s = torch.zeros_like(f), torch.zeros_like(f)
        idx = (live & (lv == l)).nonzero().squeeze(1)
        sc = 1.0 / strides[l]
        for run in _chunks(idx, rois, out, sc, sampling_ratio, (C * H * W, 8 * C * out * out)):
            y = orh.roi_align(f, rois[run], out, sc, sampling_ratio)
            if not y.requires_grad:                  # every RoI of the run has an empty sample grid
                continue
            g +=torch.autograd.grad(y, f, grad_y[run], retain_graph=True)[0]
            s += torch.autograd.grad(y, f, grad_y[run].abs())[0]
        res.append((g.permute(0, 2, 3, 1), s.permute(0, 2, 3, 1), counts[l]))
    return res


def bbox2delta_f32(p, g, means, stds):
    """box_coder.cuh bbox2delta in fp32, one rounding per operation; the logs correctly rounded.  p, g (n, 4) -> (n, 4) fp32"""
    p, g = np.asarray(p, np.float32), np.asarray(g, np.float32)
    h = np.float32(0.5)
    px, py = (p[:, 0] + p[:, 2]) * h, (p[:, 1] + p[:, 3]) * h
    pw, ph = p[:, 2] - p[:, 0], p[:, 3] - p[:, 1]
    gx, gy = (g[:, 0] + g[:, 2]) * h, (g[:, 1] + g[:, 3]) * h
    gw, gh = g[:, 2] - g[:, 0], g[:, 3] - g[:, 1]
    with np.errstate(divide='ignore', invalid='ignore'):
        d = [(gx - px) / pw, (gy - py) / ph, np.log((gw / pw).astype(np.float64)).astype(np.float32),
             np.log((gh / ph).astype(np.float64)).astype(np.float32)]
    m, s = np.asarray(means, np.float32), np.asarray(stds, np.float32)
    return np.stack([(d[k] - m[k]) / s[k] for k in range(4)], 1)


def ulp_diff(a, b):
    """distance in fp32 ulps between two fp32 arrays of finite values"""
    def ordered(x):
        i = np.asarray(x, np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7fffffff), i)
    return np.abs(ordered(a) - ordered(b))


def argmax_rule(x):
    """the accuracy's predicted column of each row: torch.argmax on the CPU (the first NaN, else the first maximum)"""
    return torch.argmax(x.cpu(), dim=1)


def accuracy_f32(x, labels):
    """ptb_roi_accuracy's value: fp32(correct) * fp32(100 / R)"""
    correct = int((argmax_rule(x) == labels.cpu()).sum())
    return np.float32(correct) * np.float32(100.0 / x.shape[0])


def decode64(rois, cls_score, bbox_pred, B, num_classes, agnostic, means, stds, max_ratio, img_hw, scale_factor=None):
    """ptb_roi_decode in float64 from the fp32 inputs: (boxes (B, N, C, 4), scores (B, N, C), M (B, N)) with M the row's largest
    intermediate magnitude (RoI coordinates, pw * dx, ph * dy, the centres gx, gy, gw, gh, H, W), divided by the row's smallest
    scale factor when rescaling"""
    rois, cls_score, bbox_pred, img_hw = rois.cpu(), cls_score.cpu(), bbox_pred.cpu(), img_hw.cpu()
    M, C = rois.shape[0], num_classes
    N = M // B
    pad = (rois[:, 1:].abs().sum(1) == 0)
    x = cls_score.double().clone()
    x[pad] = 0
    scores = torch.softmax(x, 1)[:, :C]
    d = bbox_pred.double().view(M, -1, 4).clone()
    d[pad] = 0
    d = d * torch.tensor(np.asarray(stds, np.float32), dtype=torch.float64) + torch.tensor(np.asarray(means, np.float32), dtype=torch.float64)
    d = d.expand(M, C, 4) if agnostic else d
    r = rois[:, 1:].double()
    px, py = ((r[:, 0] + r[:, 2]) * 0.5)[:, None], ((r[:, 1] + r[:, 3]) * 0.5)[:, None]
    pw, ph = (r[:, 2] - r[:, 0])[:, None], (r[:, 3] - r[:, 1])[:, None]
    mr = float(np.float32(max_ratio))
    dw, dh = d[..., 2].clamp(-mr, mr), d[..., 3].clamp(-mr, mr)
    gw, gh = pw * dw.exp(), ph * dh.exp()
    gx, gy = px + pw * d[..., 0], py + ph * d[..., 1]
    b = torch.stack([gx - gw * 0.5, gy - gh * 0.5, gx + gw * 0.5, gy + gh * 0.5], -1)
    hw = img_hw.double().repeat_interleave(N, 0)                     # (M, 2) per row
    lim = torch.stack([hw[:, 1], hw[:, 0], hw[:, 1], hw[:, 0]], -1)[:, None, :]
    b = torch.minimum(torch.clamp(b, min=0.0), lim)
    mag = torch.stack([r.abs().amax(1), (pw * d[..., 0]).abs().amax(1), (ph * d[..., 1]).abs().amax(1), gx.abs().amax(1),
                       gy.abs().amax(1), gw.abs().amax(1), gh.abs().amax(1), hw.amax(1)], 1).amax(1)
    if scale_factor is not None:
        sf = scale_factor.cpu().double().repeat_interleave(N, 0)      # (M, 4)
        b = b / sf[:, None, :]
        mag = mag / sf.amin(1)
    return b.view(B, N, C, 4), scores.view(B, N, C), mag.view(B, N)


def bbox_loss64(bbox_pred, labels, bbox_targets, bbox_weights, num_classes, agnostic, smooth, beta):
    """RoIBoxLoss in float64 over the positive rows (0 <= label < num_classes): (sum, d sum / d bbox_pred (R, ld), the mask of the
    columns the loss reads)"""
    p64 = bbox_pred.detach().cpu().double().requires_grad_(True)
    lab = labels.cpu()
    R = p64.shape[0]
    pos = ((lab >= 0) & (lab < num_classes)).nonzero().squeeze(1)
    cols = torch.arange(4)[None, :] + (0 if agnostic else 4 * lab[pos][:, None])
    pred = p64[pos[:, None], cols]
    d = pred - bbox_targets.cpu().double()[pos]
    a = d.abs()
    if smooth:
        b = float(np.float32(beta))
        l = torch.where(a < b, 0.5 * a * a / b, a - 0.5 * b)
    else:
        l = a
    s = (l * bbox_weights.cpu().double()[pos]).sum()
    s.backward()
    read = torch.zeros(R, p64.shape[1], dtype=torch.bool)
    read[pos[:, None], cols] = True
    return float(s.detach()), p64.grad, read
