"""Host restatement of the chunked MIL forward (csrc/mil.cu, mil_fwd_kernel above 256 classes) and float64 references of the MIL and
AllPos bag losses as functions of the bag logits (test infrastructure, CPU).

mil_fwd_chunked restates the kernel's reduction order in fp32 numpy:
  * per (bag, class): slice s in 0..3 sums the samples k = s, s + 4, ... in order (max, then Z, T, N), the slices merge in order 0..3;
  * the classes are walked in chunks of `cp` lanes; slice 0 forms the chunk's loss terms, each warp adds its 32 lanes by the xor butterfly
    of warp_sum, and thread 0 adds the warp sums to the bag's running total in class order;
  * top-1 class: the lanes' (probability, class) pairs reduce with "larger wins, equal -> smaller class", merged across chunks the same way.
The per-(bag, class) values do not depend on the chunk width; only the bag loss sum does (through the warp order, not the chunking of a
class).  exp / log are numpy's fp32 functions, not CUDA's, so the restatement fixes the order, not the last bits of the GPU's result."""
import numpy as np
import torch

from oracle import cpr as ocpr
from tests.cpr_loss_types_ref import bce

MIL_KS = 4
MIL_MAXCP = 256


def mil_lanes(C):
    """class lanes per chunk of ptb_mil_loss_fwd / _bwd: C rounded up to a warp, at most 256."""
    return min((C + 31) // 32 * 32, MIL_MAXCP)


def _term(p, q, lw, eps, kind):
    p, q = np.float32(p), np.float32(q)
    if kind == 0:
        l1 = (p - q) * (p - q)
        l2 = q * np.log(p + np.float32(eps)) + (np.float32(1) - q) * np.log(np.float32(1) - p + np.float32(eps))
        return np.float32(-(l1 * l2)) * np.float32(lw)
    return np.float32((q - 1) * max(np.log1p(-p), np.float32(-100)) - q * max(np.log(p) if p > 0 else np.float32(-np.inf), np.float32(-100)))


def _warp_sum(v):
    v = v.astype(np.float32).copy()
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = (v + v[lanes ^ o]).astype(np.float32)
    return v[0]


def mil_fwd_chunked(bl, N, NP, weight, labels, eps, kind, cp=None):
    """bl (G,K,LD), weight (G,K), labels (G,) -> prob (G,N) fp32, bag loss (G,) fp32, label weight (G,), top-1 class (G,)."""
    bl = np.asarray(bl, dtype=np.float32)
    weight = np.asarray(weight, dtype=np.float32)
    G, K, _ = bl.shape
    cp = cp or mil_lanes(N)
    prob = np.zeros((G, N), np.float32)
    loss = np.zeros(G, np.float32)
    lw = (weight.sum(axis=1) > 0).astype(np.float32)
    top = np.zeros(G, np.int64)
    with np.errstate(over='ignore', divide='ignore', invalid='ignore'):
        for g in range(G):
            cls, ins, w = bl[g, :, :N], bl[g, :, NP:NP + N], weight[g]
            sig = (np.float32(1) / (np.float32(1) + np.exp(-cls))).astype(np.float32)
            mx = np.full(N, -np.inf, np.float32)
            for s in range(MIL_KS):
                for k in range(s, K, MIL_KS):
                    mx = np.maximum(mx, ins[k])
            z, t, n = (np.zeros(N, np.float32) for _ in range(3))
            for s in range(MIL_KS):
                zs, ts, ns = (np.zeros(N, np.float32) for _ in range(3))
                for k in range(s, K, MIL_KS):
                    e = np.exp(ins[k] - mx).astype(np.float32)
                    zs = (zs + e).astype(np.float32)
                    ts = (ts + e * w[k]).astype(np.float32)
                    ns = (ns + sig[k] * (e * w[k])).astype(np.float32)
                z, t, n = (z + zs).astype(np.float32), (t + ts).astype(np.float32), (n + ns).astype(np.float32)
            tn = (t / z).astype(np.float32)
            prob[g] = ((n / z) / np.maximum(tn, np.float32(1e-12))).astype(np.float32)
            tot, best, besti = np.float32(0), np.float32(-np.inf), np.iinfo(np.int64).max
            for c0 in range(0, N, cp):
                lanes = np.arange(c0, c0 + cp)
                act = lanes < N
                terms = np.array([_term(prob[g, c], 1.0 if c == labels[g] else 0.0, lw[g], eps, kind) if a else np.float32(0)
                                  for c, a in zip(lanes, act)], np.float32)
                for w0 in range(0, cp, 32):
                    tot = np.float32(tot + _warp_sum(terms[w0:w0 + 32]))
                    for c in lanes[w0:w0 + 32][act[w0:w0 + 32]]:
                        v = prob[g, c]
                        if v > best or (v == best and c < besti):
                            best, besti = v, c
            loss[g] = tot
            top[g] = besti
    return prob, loss, lw, top


def mil_ref64(bl, N, NP, weight, labels, eps, kind):
    """float64 MILLoss (oracle.cpr.mil_bag_prob + gfocal x label weight, or unweighted BCE) of bag logits (G,K,LD): prob (G,N), sum,
    count (#bags with weight), hits, top-two margin (G,), grad (G,K,LD) = d sum / d bl."""
    x = bl.detach().cpu().double().clone().requires_grad_(True)
    w = weight.detach().cpu().double()
    labels = labels.detach().cpu().long()
    G = x.shape[0]
    onehot = torch.zeros((G, N), dtype=torch.float64)
    onehot[torch.arange(G), labels] = 1.0
    prob = ocpr.mil_bag_prob(x[..., :N].sigmoid(), x[..., NP:NP + N], w[..., None])
    lw = (w.sum(dim=1) > 0).double()
    s = ocpr.gfocal_loss(prob, onehot, lw[:, None], eps).sum() if kind == 0 else bce(prob, onehot).sum()
    s.backward()
    p = prob.detach()
    top = p.topk(min(2, N), dim=1)[0]
    margin = (top[:, 0] - top[:, 1]) if N > 1 else torch.full((G,), float('inf'), dtype=torch.float64)
    return dict(prob=p, sum=float(s.detach()), count=float(lw.sum()), hits=float((p.argmax(dim=1) == labels).sum()), margin=margin,
                grad=x.grad)


def allpos_ref64(bl, N, weight, labels, eps, kind):
    """float64 AllPosLoss of bag logits (G,K,LD): sum (gfocal x sample weight, or unweighted BCE), count (#samples with weight > 0),
    hits (#samples whose first-maximum class is the label), top-two margin per sample."""
    p = bl[..., :N].detach().cpu().double().sigmoid()
    G, K, _ = p.shape
    w = weight.detach().cpu().double().reshape(G * K, 1)
    lab = labels.detach().cpu().long().repeat_interleave(K)
    p = p.reshape(G * K, N)
    oh = torch.zeros_like(p)
    oh[torch.arange(G * K), lab] = 1.0
    s = ocpr.gfocal_loss(p, oh, w, eps).sum() if kind == 0 else bce(p, oh).sum()
    top = p.topk(min(2, N), dim=1)[0]
    margin = (top[:, 0] - top[:, 1]) if N > 1 else torch.full((G * K,), float('inf'), dtype=torch.float64)
    return dict(sum=float(s), count=float((w > 0).sum()), hits=float((p.argmax(dim=1) == lab).sum()), margin=margin)
