"""Host restatement of the point refinement, ptb_cpr_refine and ptb_cpr_refine_fused (csrc/refine.cu), for its tests.  Plain torch on
the CPU (the fused form's logit gather may run on the map's device).

Per bag sample (refine_single, cpr_head.py:780-850) the kernels decide in fp32:
    merge_valid = valid & nearest & classify & (p > merge_th) & (p > fl(p_centre * gt_alpha)) & inside
  * valid: the point lies inside the padded image (point_valid), inside: inside img_hw;
  * classify: the FIRST maximum of the sample's class probabilities is the GT's label;
  * nearest: among the centres of the GTs with the same (image, label), in ascending GT order, the FIRST nearest one is the sample's
    own; cdist_mm or cdist_direct (ptb_common.cuh) by torch.cdist's rule, restated here with a true fma and a correctly rounded sqrt;
  * p is the label's probability, p_centre that of the centre sample (the last one of refine 0).
The fused form computes p from logits it samples from the map: gather_f32 reproduces those bit for bit and torch.sigmoid on the CPU is
the kernels' sigmoid bit for bit, so every decision above is exact here.

Per GT the kernels then add pm = merge_valid ? p : 0 in fp32 in their own order.  Here the sums are float64 and every GT carries the
error bound of its operation count, gamma(n) * sum |terms| (Higham): the mean score S / count within gamma(n + 1) * score, the mean
point sum x p / (S + 1e-8) within gamma(2n + 2) * sum |x| p / (S + 1e-8).  not_refine = score < refine_th is exact wherever the
score is further than its bound from refine_th (the others are `undecided`); a GT that is not refined returns its centre sample exactly;
in max mode the score is the exact maximum of pm, or fl(refine_th * 0.5) when that is 0.

expected_plan mirrors the fused kernel's host dispatch (class phase, TMA staging, block size, passes per warp)."""
import math
from typing import NamedTuple, Optional

import numpy as np
import torch

from tests.gather_ref import fma_f32, gather_f32, point_valid, sample_points, window_size

U = 2.0 ** -24
TAIL_LIMIT = 48 * 1024         # the fused kernel's per-sample arrays (and the stage kernel's) must fit the default shared memory
TMA_SMEM_LIMIT = 112 * 1024    # window + tail + alignment slack of the staged fused kernel: two CTAs per SM
GCAP = 256                     # group members the fused kernel holds in shared memory
EPS = float(np.float32(1e-8))


class Cfg(NamedTuple):
    merge_th: float
    gt_alpha: float
    refine_th: float
    nearest: bool
    classify: bool
    score_max: bool


def gamma(n):
    return n * U / (1 - n * U)


def f32(x):
    return float(np.float32(x))


def _r(x):
    """float64 tensor -> the same values rounded to fp32, as float64"""
    return x.float().double()


# ----------------------------------------------------------------------------------------------------------------------------------
# distances (ptb_common.cuh).  Inputs are float64 tensors holding fp32 values; a +, -, * of two fp32 values or a sqrt of one rounded to
# float64 and then to fp32 is the correctly rounded fp32 result.
# ----------------------------------------------------------------------------------------------------------------------------------
def sq_norm2(x, y):
    return _r(_r(x * x) + _r(y * y))


def cdist_direct(px, py, cx, cy):
    dx, dy = _r(px - cx).abs(), _r(py - cy).abs()
    return _r(torch.sqrt(_r(_r(dx * dx) + _r(dy * dy))))


def cdist_mm(px, py, cx, cy):
    acc = _r((-2.0 * px) * cx)
    acc = fma_f32((-2.0 * py).float(), cy.float(), acc.float()).double()
    acc = _r(acc + sq_norm2(px, py))
    acc = _r(acc + sq_norm2(cx, cy))
    return _r(torch.sqrt(acc.clamp(min=0.0)))


def use_mm(t, R, K):
    """torch.cdist's choice for t*R*K points against t*R centres"""
    return t * R * K > 25 or t * R > 25


def nearest_choice(pts, members, R, K, mm):
    """pts (G,Kt,2) fp32; members: ascending GT indices of one group.  -> (t,Kt) int64 first nearest candidate (j * R + r) of every
    sample of the members, and the (t,Kt,t*R) float64 distances"""
    t, Kt = len(members), pts.shape[1]
    P = pts[members].reshape(-1, 2).double()
    C = pts[members][:, K - 1::K][:, :R].reshape(-1, 2).double()        # centre of refine r of member j: sample r * K + K - 1
    f = cdist_mm if mm else cdist_direct
    d = f(P[:, 0:1], P[:, 1:2], C[None, :, 0], C[None, :, 1])
    first = (d == d.min(1, keepdim=True)[0]).int().argmax(1)            # argmax keeps the first of equal values
    return first.reshape(t, Kt), d.reshape(t, Kt, t * R)


def groups(bag_img, labels):
    """same-(image, label) groups in ascending GT order: a list of int64 index tensors"""
    key = bag_img.cpu().long() * (1 << 20) + labels.cpu().long()
    order = torch.argsort(key, stable=True)
    _, counts = torch.unique_consecutive(key[order], return_counts=True)
    return list(torch.split(order, counts.tolist()))


# ----------------------------------------------------------------------------------------------------------------------------------
# per-sample decisions
# ----------------------------------------------------------------------------------------------------------------------------------
class Comp(NamedTuple):
    pts: torch.Tensor        # (G,Kt,2) fp32 sample points
    pl: torch.Tensor         # (G,Kt) fp32 probability of the label
    valid: torch.Tensor      # (G,Kt) bool
    inside: torch.Tensor
    classify: torch.Tensor
    nearest: torch.Tensor    # True for every sample of a GT alone in its group
    d_own: torch.Tensor      # (G,Kt) float64 distance to the own centre, inf for a GT alone
    d_alt: torch.Tensor      # nearest other candidate
    t: torch.Tensor          # (G,) group size
    mm: torch.Tensor         # (G,) the group uses cdist_mm
    K: int


def components(prob, pts, valid, K, labels, bag_img, img_hw):
    """prob (G,Kt,C) fp32 probabilities, pts (G,Kt,2+) fp32, valid (G,Kt) bool, Kt = R * K with the centre of refine r at r * K + K - 1,
    labels / bag_img (G,), img_hw (B,2) int."""
    prob, valid = prob.cpu().float(), valid.cpu().bool()
    pts = pts.cpu().float()[..., :2].contiguous()
    G, Kt, C = prob.shape
    R = Kt // K
    lab = labels.cpu().long()
    pl = prob.gather(2, lab[:, None, None].expand(G, Kt, 1))[..., 0]
    pmax = prob.max(2)[0]
    classify = torch.empty((G, Kt), dtype=torch.bool)
    cls_idx = torch.arange(C)
    for j in range(0, G, max(1, (1 << 22) // max(1, Kt * C))):
        sl = slice(j, j + max(1, (1 << 22) // max(1, Kt * C)))
        below = cls_idx[None, None, :] < lab[sl, None, None]
        classify[sl] = (pl[sl] == pmax[sl]) & ~((prob[sl] == pl[sl, :, None]) & below).any(2)
    hw = img_hw.cpu()[bag_img.cpu().long()].float()
    x, y = pts[..., 0], pts[..., 1]
    inside = (x < hw[:, 1:2]) & (x >= 0) & (y < hw[:, 0:1]) & (y >= 0)
    nearest = torch.ones((G, Kt), dtype=torch.bool)
    d_own = torch.full((G, Kt), math.inf, dtype=torch.float64)
    d_alt = torch.full((G, Kt), math.inf, dtype=torch.float64)
    tt = torch.ones(G, dtype=torch.int64)
    mm = torch.zeros(G, dtype=torch.bool)
    for members in groups(bag_img, labels):
        t = len(members)
        tt[members] = t
        if t < 2:
            continue
        m = use_mm(t, R, K)
        mm[members] = m
        first, d = nearest_choice(pts, members, R, K, m)
        own = torch.arange(t)[:, None] * R + torch.arange(Kt)[None, :] // K
        nearest[members] = first == own
        do = d.gather(2, own[..., None])[..., 0]
        d_own[members] = do
        d_alt[members] = d.scatter(2, own[..., None], math.inf).min(2)[0]
    return Comp(pts, pl, valid, inside, classify, nearest, d_own, d_alt, tt, mm, K)


def fused_components(lmap, ncls, centers, labels, bag_img, offsets, stride, pad_hw, img_hw):
    """components of ptb_cpr_refine_fused's inputs: logits by gather_f32 (on lmap's device), probabilities by CPU torch.sigmoid"""
    logits = gather_f32(lmap, centers, bag_img, offsets, stride, C=ncls).cpu()
    pts = sample_points(centers.cpu(), offsets.cpu())
    valid = point_valid(centers.cpu(), bag_img.cpu(), offsets.cpu(), pad_hw.cpu())
    return components(torch.sigmoid(logits), pts, valid, offsets.shape[0], labels, bag_img, img_hw)


# ----------------------------------------------------------------------------------------------------------------------------------
# per-GT reduction
# ----------------------------------------------------------------------------------------------------------------------------------
class Ref(NamedTuple):
    merge_valid: torch.Tensor   # (G,Kt) bool
    chosen: torch.Tensor        # (G,Kt) bool
    not_refine: torch.Tensor    # (G,) bool; the kernel's value where not undecided
    undecided: torch.Tensor     # (G,) bool: |score - refine_th| within the score's bound, not_refine_in not set
    score: torch.Tensor         # (G,) float64: exact mean score, or in max mode the exact fp32 output
    score_bound: torch.Tensor   # (G,) float64 (0 in max mode)
    mean: torch.Tensor          # (G,2) float64 weighted mean point
    mean_bound: torch.Tensor    # (G,2) float64
    centre: torch.Tensor        # (G,2) fp32: the point of a GT that is not refined


def combine(comp, cfg, not_refine_in=None):
    K = comp.K
    Kt = comp.pl.shape[1]
    m = comp.valid & comp.inside
    if cfg.nearest:
        m = m & comp.nearest
    if cfg.classify:
        m = m & comp.classify
    pl = comp.pl
    pga = (pl[:, K - 1].double() * f32(cfg.gt_alpha)).float()           # one fp32 product
    m = m & (pl > f32(cfg.merge_th)) & (pl > pga[:, None])
    pm = torch.where(m, pl, torch.zeros_like(pl))
    p = pm.double()
    S = p.sum(1)
    cnt = (pm > 0).sum(1).double()
    score = torch.where(cnt > 0, S / cnt.clamp(min=1), torch.zeros_like(S))
    score_bound = gamma(Kt + 1) * score
    th = f32(cfg.refine_th)
    nr = score < th
    undecided = (score - th).abs() <= score_bound
    if not_refine_in is not None:
        nr_in = not_refine_in.cpu().bool()
        nr = nr | nr_in
        undecided = undecided & ~nr_in
    xy = comp.pts.double()
    mean = (xy * p[..., None]).sum(1) / (S + EPS)[:, None]
    mean_bound = gamma(2 * Kt + 2) * (xy.abs() * p[..., None]).sum(1) / (S + EPS)[:, None]
    if cfg.score_max:
        mx = pm.max(1)[0]
        score = torch.where(mx == 0, torch.full_like(mx, float(np.float32(th) * np.float32(0.5))), mx).double()
        score_bound = torch.zeros_like(score)
    return Ref(m, pm > 0, nr, undecided, score, score_bound, mean, mean_bound, comp.pts[:, K - 1])


def refine_ref(prob, pts, valid, K, labels, bag_img, img_hw, cfg, not_refine_in=None):
    return combine(components(prob, pts, valid, K, labels, bag_img, img_hw), cfg, not_refine_in)


def check(ref, pts, score, not_refine, chosen=None, merge_valid=None):
    """compares a kernel's outputs with the reference; returns (list of failures, worst float error / bound, #undecided GTs)"""
    pts, score, nr = pts.cpu(), score.cpu(), not_refine.cpu().bool()
    bad = []
    if chosen is not None and not torch.equal(chosen.cpu().bool(), ref.chosen):
        bad.append(f'chosen: {int((chosen.cpu().bool() != ref.chosen).sum())} samples differ')
    if merge_valid is not None and not torch.equal(merge_valid.cpu().bool(), ref.merge_valid):
        bad.append(f'merge_valid: {int((merge_valid.cpu().bool() != ref.merge_valid).sum())} samples differ')
    dec = ~ref.undecided
    if not torch.equal(nr[dec], ref.not_refine[dec]):
        bad.append(f'not_refine: {int((nr[dec] != ref.not_refine[dec]).sum())} decided GTs differ')
    worst = 0.0
    if nr.any() and not torch.equal(pts[nr], ref.centre[nr]):
        bad.append(f'points of GTs not refined: {int((pts[nr] != ref.centre[nr]).any(1).sum())} are not the centre sample')
    keep = ~nr
    if keep.any():
        err = (pts[keep].double() - ref.mean[keep]).abs()
        bnd = ref.mean_bound[keep]
        if (err > bnd).any():
            bad.append(f'refined points: {int((err > bnd).any(1).sum())} outside the bound')
        worst = max(worst, float((err / bnd.clamp(min=1e-300)).max()))
    serr = (score.double() - ref.score).abs()
    if (serr > ref.score_bound).any():
        bad.append(f'scores: {int((serr > ref.score_bound).sum())} outside the bound')
    pos = ref.score_bound > 0
    if pos.any():
        worst = max(worst, float((serr[pos] / ref.score_bound[pos]).max()))
    return bad, worst, int(ref.undecided.sum())


# ----------------------------------------------------------------------------------------------------------------------------------
# dispatch (ptb_cpr_refine_fused host code)
# ----------------------------------------------------------------------------------------------------------------------------------
class Plan(NamedTuple):
    phase: str                  # 'fast<1>'..'fast<4>' (rf_class_phase<NT>) or 'loop' (rf_class_phase_loop)
    use_tma: bool               # the window is staged by TMA (bags that straddle it still read global memory)
    fallback: Optional[str]     # why not: 'env' (PTB_REFINE_TMA=0), 'reach0', 'ld' (> 256), 'window' (> 112 KB)
    ws: int                     # window side in cells (0 when not computed)
    threads: int
    passes: int                 # 32-sample passes of warp 0


def class_phase(ncls):
    cg4 = (ncls + 3) // 4
    nt = (cg4 + 7) // 8
    return f'fast<{nt}>' if ncls % 4 == 0 and nt <= 4 else 'loop'


def tail_bytes(K):
    return 16 * K + (K + 15) // 16 * 16


def expected_plan(ncls, ld, K, reach_px, stride, env):
    """env holds PTB_REFINE_TMA.  Assumes the tensor map encodes (it does for every layout the host accepts).  Raises ValueError where
    the host refuses the bag size."""
    tail = tail_bytes(K)
    if tail > TAIL_LIMIT:
        raise ValueError('bag too large for shared memory')
    warps = min(max((K + 31) // 32, 2), 10)
    passes = -(-K // (32 * warps))
    phase = class_phase(ncls)
    e = env.get('PTB_REFINE_TMA')
    reach = f32(reach_px)
    ws = 0
    if e is not None and e[:1] == '0':
        fallback = 'env'
    elif not reach > 0:
        fallback = 'reach0'
    elif ld > 256:
        fallback = 'ld'
    else:
        ws = window_size(reach, stride)
        if ws <= 256 and ws * ws * ld * 4 + tail + 128 <= TMA_SMEM_LIMIT:
            return Plan(phase, True, None, ws, warps * 32, passes)
        fallback = 'window'
    return Plan(phase, False, fallback, ws, warps * 32, passes)
