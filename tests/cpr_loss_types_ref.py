"""float64 reference of the positive-bag loss kinds (MILLoss gfocal / binary_cross_entropy, AllPosLoss gfocal / binary_cross_entropy) as
a function of the [cls | ins] logit map or of sampled bag logits (test infrastructure, CPU).

The BCE term is restated from ATen's CPU formula (aten/src/ATen/native/Loss.cpp), not called, so that its float64 values can be pinned
against torch.nn.functional.binary_cross_entropy:
  value(p, t) = (t - 1) * max(log1p(-p), -100) - t * max(log p, -100),   d/dp = (p - t) / max((1 - p) p, 1e-12 in fp32).
The sample geometry (taps, validity) is tests/cpr_loss_ref.py's.
"""
import numpy as np
import torch

from oracle import cpr as ocpr
from tests.cpr_loss_ref import point_valid, taps


BCE_GRAD_EPS = float(np.float32(1e-12))      # ATen's EPSILON is a float constant: 1e-12 rounded to fp32, also in float64 backward


class _Bce(torch.autograd.Function):
    @staticmethod
    def forward(ctx, p, t):
        ctx.save_for_backward(p, t)
        return (t - 1) * torch.clamp(torch.log1p(-p), min=-100.0) - t * torch.clamp(torch.log(p), min=-100.0)

    @staticmethod
    def backward(ctx, g):
        p, t = ctx.saved_tensors
        return g * (p - t) / torch.clamp((1 - p) * p, min=BCE_GRAD_EPS), None


def bce(p, t):
    """elementwise binary cross-entropy with ATen's clamps and ATen's (clamped) derivative."""
    return _Bce.apply(p, t)


def term(p, t, w, eps, kind):
    """per-element loss: gfocal x w (kind 0) or unweighted BCE (kind 1)."""
    if kind == 0:
        return -(((p - t) ** 2) * (t * (p + eps).log() + (1 - t) * (1 - p + eps).log()) * w)
    return bce(p, t)


def mil_from_bag_logits(bl, N, NP, weight, labels, eps, kind):
    """MILLoss on sampled rows (G,K,LD) f64 with weights (G,K): returns loss sum, #bags with weight, #hits, bag prob (G,N)."""
    G = bl.shape[0]
    prob = ocpr.mil_bag_prob(bl[..., :N].sigmoid(), bl[..., NP:NP + N], weight[..., None])
    lw = (weight.sum(dim=1) > 0).double()
    onehot = torch.zeros((G, N), dtype=torch.float64)
    onehot[torch.arange(G), labels] = 1.0
    s = term(prob, onehot, lw[:, None], eps, kind).sum()
    hit = prob.detach().argmax(dim=1) == labels
    return s, float(lw.sum()), float(hit.sum()), prob


def allpos_from_bag_logits(bl, N, weight, labels, eps, kind):
    """AllPosLoss on sampled rows: returns loss sum, #samples with weight > 0, #samples whose top-1 class is the label, probs (G,K,N)."""
    G, K = weight.shape
    prob = bl[..., :N].sigmoid()
    onehot = torch.zeros((G, K, N), dtype=torch.float64)
    onehot[torch.arange(G)[:, None], torch.arange(K)[None, :], labels[:, None]] = 1.0
    s = term(prob, onehot, weight[..., None], eps, kind).sum()
    hit = prob.detach().argmax(dim=-1) == labels[:, None]
    return s, float((weight > 0).sum()), float(hit.sum()), prob


def loss_map_ref(lmap, N, NP, centers, bag_img, offsets, stride, pad_hw, labels, eps, allpos, kind, scale_pos=1.0, scale_gt=0.0):
    """float64 positive-bag loss (+ gt term) as a function of the logit map and its gradient d total / d lmap (B,H,W,LD)."""
    B, H, W, LD = lmap.shape
    K = offsets.shape[0]
    L = lmap.detach().cpu().double().reshape(B * H * W, LD).clone().requires_grad_(True)
    centers, bag_img, offsets, labels = centers.cpu(), bag_img.cpu(), offsets.cpu(), labels.cpu().long()
    idx, w = taps(centers, bag_img, offsets, stride, H, W)
    bl = (L[idx] * w[..., None]).sum(dim=2)
    weight = point_valid(centers, bag_img, offsets, pad_hw.cpu()).double()
    if allpos:
        s, cnt, hits, prob = allpos_from_bag_logits(bl, N, weight, labels, eps, kind)
    else:
        s, cnt, hits, prob = mil_from_bag_logits(bl, N, NP, weight, labels, eps, kind)
    G = centers.shape[0]
    onehot = torch.zeros((G, N), dtype=torch.float64)
    onehot[torch.arange(G), labels] = 1.0
    gt_sum = ocpr.gfocal_loss(bl[:, K - 1, :N].sigmoid(), onehot, weight[:, K - 1:K], eps).sum()
    total = scale_pos * s + scale_gt * gt_sum
    total.backward()
    return dict(sum=s.detach(), count=cnt, hits=hits, prob=prob.detach(), weight=weight, grad=L.grad.reshape(B, H, W, LD))
