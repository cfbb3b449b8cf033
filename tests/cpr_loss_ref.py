"""float64 reference of the fused CPR training loss as a function of the [cls | ins] logit map (test infrastructure, CPU).

The loss kernels (ptb_cpr_bag_mil_fwd, ptb_mil_loss_fwd, ptb_gfocal_sigmoid_fwd, ptb_sigmoid_loss_bwd, ptb_cpr_loss_bwd_map, ptb_cpr_loss_bwd_scatter) see
the head only through its logit map lmap (B,H,W,LD): class logits in columns [0, N), instance logits in [NP, NP+N), padding elsewhere.
This module restates what they compute from that map:

  * sample positions in fp32 with the kernels' operation order (sample_coord / make_taps in csrc/ptb_common.cuh, which is also ATen's
    fp32 unnormalize + border clamp of grid_sample): p = offset + centre, u = p / stride, g = (2u + 1) / size - 1,
    ix = fma(g + 1, size / 2, -0.5), clamped to [0, size - 1];
  * bilinear weights and everything after them in float64, so the reference is exact arithmetic at the kernels' own sample points;
  * the loss terms with the oracle's functions (oracle.cpr.mil_bag_prob, gfocal_loss: MILLoss and the gt / neg gfocal terms of
    CPRHead.loss0), and d loss / d lmap from float64 autograd.

The fp32 rounding of the sample position is reproduced in float64: +, *, / of two fp32 values rounded once to fp32 is the correctly
rounded fp32 result, and the fma's product (g + 1) * size / 2 has at most 36 significant bits, so adding -0.5 is exact in float64
whenever the result is >= 0 (negative results are clamped to 0 on both sides).
"""
import numpy as np
import torch

from oracle import cpr as ocpr


def _f32(x):
    return x.float().double()


def sample_coord(p, stride, size):
    """fp32 sample coordinate of image coordinate p (fp32 tensor) along an axis of `size` cells -> float64 tensor holding fp32 values."""
    p = p.double()
    u = _f32(p / float(np.float32(stride)))
    t = _f32(_f32(2.0 * u) + 1.0)
    g = _f32(_f32(t / float(size)) - 1.0)
    ix = _f32((_f32(g + 1.0) * (0.5 * float(size))) - 0.5)
    return ix.clamp(min=0.0, max=float(size - 1))


def sample_points(centers, offsets):
    """(G,2), (K,2) fp32 -> (G,K,2) fp32 image coordinates (offset + centre, one fp32 add: cpr_head.py:492-497)."""
    return offsets.float()[None, :, :] + centers.float()[:, None, :]


def taps(centers, bag_img, offsets, stride, H, W):
    """cell index (into the (B*H*W) rows of the map) and float64 weight of the four taps of every sample: (G,K,4) int64, (G,K,4) f64."""
    pts = sample_points(centers, offsets)
    ix = sample_coord(pts[..., 0], stride, W)
    iy = sample_coord(pts[..., 1], stride, H)
    x0, y0 = ix.floor(), iy.floor()
    x1, y1 = (x0 + 1).clamp(max=W - 1), (y0 + 1).clamp(max=H - 1)          # a clamped east / south tap has weight 0
    wx, wy = ix - x0, iy - y0
    ex, ey = 1.0 - wx, 1.0 - wy
    base = bag_img.long()[:, None] * (H * W)
    idx = torch.stack([base + (y0 * W + x0).long(), base + (y0 * W + x1).long(), base + (y1 * W + x0).long(),
                       base + (y1 * W + x1).long()], dim=-1)
    w = torch.stack([ex * ey, wx * ey, ex * wy, wx * wy], dim=-1)
    return idx, w


def point_valid(centers, bag_img, offsets, pad_hw):
    """(G,K) bool: 0 <= x < pad_w and 0 <= y < pad_h (cpr_head.py:172-180) on the fp32 sample points."""
    pts = sample_points(centers, offsets)
    ph = pad_hw[bag_img.long(), 0].float()[:, None]
    pw = pad_hw[bag_img.long(), 1].float()[:, None]
    return ocpr.point_valid(pts, ph, pw)


def oracle_bag_logits(lmap, centers, bag_img, offsets, stride):
    """the oracle's fp32 bag logits (G,K,LD): oracle.cpr.sample_point_feat (F.grid_sample, border padding) image by image.
    The kernels' sampled logits must equal these bit for bit."""
    B, H, W, LD = lmap.shape
    out = torch.zeros((centers.shape[0], offsets.shape[0], LD), dtype=torch.float32)
    pts = sample_points(centers, offsets)
    for b in range(B):
        sel = (bag_img.long() == b).nonzero().flatten()
        if len(sel):
            out[sel] = ocpr.sample_point_feat(lmap[b:b + 1].permute(0, 3, 1, 2).float(), pts[sel], stride)
    return out


def cpr_loss_ref(lmap, N, NP, centers, bag_img, offsets, stride, pad_hw, labels, eps, scale_mil=0.0, scale_gt=0.0, scale_neg=0.0,
                 neg_mask=None, with_mil=True, want_grad=True):
    """float64 forward (and backward) of the loss as a function of the logit map.

    lmap (B,H,W,LD) fp32; centers (G,2) fp32; bag_img (G,) int; offsets (K,2) fp32, centre sample LAST; pad_hw (B,2) int; labels (G,) int;
    neg_mask (B,H,W,N) 0/1 or None.  The three scales multiply the un-normalised loss sums (the head divides them by its counts).
    Returns a dict:
      bag_logits (G,K,LD) f64, weight (G,K) f64 0/1, valid_center (G,) f64,
      bag_prob (G,N), mil_sum, label_weight (G,), stats = (#bags with weight, #top-1 hits), top_margin (G,) = top-1 minus top-2 bag
      probability (inf for one class), hit (G,) bool,
      mt_max (G,N) = max over the bag of the fp32 sampled instance logits (the forward kernels' exact maximum), inv_t (G,N) = 1/T with
      T = sum_k exp(ins_k - mt_max) * w_k (0 where the F.normalize clamp is active, as the kernels store it),
      gt_sum, neg_sum, total = scale_mil * mil_sum + scale_gt * gt_sum + scale_neg * neg_sum,
      grad (B,H,W,LD) f64 = d total / d lmap (when want_grad)."""
    B, H, W, LD = lmap.shape
    G, K = centers.shape[0], offsets.shape[0]
    L = lmap.detach().cpu().double().reshape(B * H * W, LD).clone().requires_grad_(want_grad)
    centers, bag_img, offsets = centers.cpu(), bag_img.cpu(), offsets.cpu()
    idx, w = taps(centers, bag_img, offsets, stride, H, W)
    bl = (L[idx] * w[..., None]).sum(dim=2)                                  # (G,K,LD)
    weight = point_valid(centers, bag_img, offsets, pad_hw.cpu()).double()
    labels = labels.cpu().long()
    onehot = torch.zeros((G, N), dtype=torch.float64)
    onehot[torch.arange(G), labels] = 1.0
    cls, ins = bl[..., :N], bl[..., NP:NP + N]
    out = dict(bag_logits=bl.detach(), weight=weight, valid_center=weight[:, K - 1])
    zero = torch.zeros((), dtype=torch.float64)
    total = zero
    if with_mil:
        prob = ocpr.mil_bag_prob(cls.sigmoid(), ins, weight[..., None])     # (G,N)
        lw = (weight.sum(dim=1) > 0).double()
        mil_sum = ocpr.gfocal_loss(prob, onehot, lw[:, None], eps).sum()
        p = prob.detach()
        top = p.topk(min(2, N), dim=1)[0]
        margin = (top[:, 0] - top[:, 1]) if N > 1 else torch.full((G,), float('inf'), dtype=torch.float64)
        hit = p.argmax(dim=1) == labels
        ins32 = oracle_bag_logits(lmap.detach().cpu(), centers, bag_img, offsets, stride)[..., NP:NP + N]
        mt_max = ins32.max(dim=1)[0].double()                                # (G,N)
        e = torch.exp(ins.detach() - mt_max[:, None, :])
        T = (e * weight[..., None]).sum(dim=1)
        Z = e.sum(dim=1)
        inv_t = torch.where(T / Z >= 1e-12, 1.0 / T, torch.zeros_like(T))
        out.update(bag_prob=p, mil_sum=mil_sum.detach(), label_weight=lw, stats=(float(lw.sum()), float(hit.sum())),
                   top_margin=margin, hit=hit, mt_max=mt_max, inv_t=inv_t)
        total = total + scale_mil * mil_sum
    gt_sum = ocpr.gfocal_loss(cls[:, K - 1].sigmoid(), onehot, weight[:, K - 1:K], eps).sum()
    out['gt_sum'] = gt_sum.detach()
    total = total + scale_gt * gt_sum
    if neg_mask is not None:
        nm = neg_mask.detach().cpu().reshape(B * H * W, N).double()
        neg_prob = L[:, :N].sigmoid()
        neg_sum = ocpr.gfocal_loss(neg_prob, torch.zeros_like(neg_prob), nm, eps).sum()
        out['neg_sum'] = neg_sum.detach()
        total = total + scale_neg * neg_sum
    out['total'] = total.detach()
    if want_grad:
        total.backward()
        out['grad'] = L.grad.reshape(B, H, W, LD)
        # sensitivity of every gradient element to the fp32 rounding of the sigmoids it is made of (see probability_sensitivity)
        kap = torch.zeros((G, K, LD), dtype=torch.float64)
        if with_mil:
            pg = prob.detach().clone().requires_grad_(True)
            gp, = torch.autograd.grad(ocpr.gfocal_loss(pg, onehot, lw[:, None], eps).sum() * scale_mil, pg)
            e = torch.exp(ins.detach() - ins.detach().max(dim=1, keepdim=True)[0]) * weight[..., None]
            pi = e / e.sum(dim=1, keepdim=True).clamp(min=1e-300)
            gpi = (gp[:, None, :] * pi).abs()                                # d grad / d sigmoid of the MIL terms (cls and ins) <= |gp pi|
            kap[..., :N] += gpi
            kap[..., NP:NP + N] += gpi
        kap[:, K - 1, :N] += probability_sensitivity(cls.detach()[:, K - 1], onehot, weight[:, K - 1:K], eps, scale_gt)
        kmap = torch.zeros((B * H * W, LD), dtype=torch.float64)
        for t in range(4):
            kmap.index_add_(0, idx[..., t].reshape(-1), (w[..., t, None] * kap).reshape(-1, LD))
        if neg_mask is not None:
            kmap[:, :N] += probability_sensitivity(L.detach()[:, :N], torch.zeros((B * H * W, N), dtype=torch.float64), nm, eps, scale_neg)
        out['kappa'] = kmap.reshape(B, H, W, LD)
    return out


def probability_sensitivity(x, q, w, eps, scale):
    """|d/dp of the gradient scale * d gfocal(p, q, w) / d x| at p = sigmoid(x), float64, elementwise.

    The kernels (and the reference model's own fp32 formula) compute p = sigmoid(x) in fp32 and then 1 - p, p + eps, 1 - p + eps from it.
    An absolute error of a few fp32 ulps of 1 in p is amplified in 1 - p when p is near 1, and in (1 - p) / (1 - p + eps) when 1 - p is
    near eps: the gradient element then moves by about (this sensitivity) x (error of p).  Tests allow that on top of their relative
    tolerance."""
    p = torch.sigmoid(x.double()).detach().requires_grad_(True)
    dl, = torch.autograd.grad(ocpr.gfocal_loss(p, q, w, eps).sum() * scale, p, create_graph=True)
    h = dl * p * (1 - p)                                                     # d loss / d x
    dh, = torch.autograd.grad(h.sum(), p)
    return dh.abs().detach()
