"""The CPR loss kernels on their own against the float64 reference of tests/cpr_loss_ref.py, across the class counts, logit row widths
and bag sizes the head dispatches on (cpr_head.loss_bwd_plan):

  tiles    ptb_cpr_bag_mil_fwd -> ptb_cpr_loss_bwd_map              NP = ceil16(N): LD = 32 .. 160, K = 1 .. 320
  scatter  ptb_cpr_bag_mil_fwd -> ptb_cpr_loss_bwd_scatter          NP = ceil8(N), N <= 128, K up to 361
           ptb_cpr_bag_gather + ptb_mil_loss_fwd -> scatter          N = 129 .. 256
  staged   ptb_mil_loss_bwd + ptb_sigmoid_loss_bwd + ptb_cpr_bag_gather_bwd

Every case runs on 3 images of 13 x 21 cells (not a multiple of the 8 x 8 tile), one of them without GTs, with centres outside the padded
image (label weight 0), exactly at (0, 0) and at the pad edge, and a duplicated centre; the pad columns of the logit map hold 50.

Tolerances.  The sampled logits and their validity are bit-exact (the same fp32 operations as F.grid_sample).  The kernels evaluate
exp / log / division with __expf, __logf and __fdividef (loss_bwd.cu, a few ulp each, relative error ~1e-6 on a gradient element) and
accumulate in fp32 (K * 4 taps per cell and class, relative ~1e-6 for K = 361, more where contributions of both signs cancel; the scatter
kernel's atomic order changes from run to run); the forward uses expf / logf.  The largest error measured on an H100 was 2.0e-5 (scatter,
N = 200).  So the gradients are held to 5e-5 and the loss sums and probabilities to 1e-5 of their scale (tests/helpers.scale_rel_err),
four and ten times tighter than the head tests (2e-4 / 1e-4).  One error source is larger and is not the kernels' doing: the gradient
is built from p = sigmoid(x) in fp32, and 1 - p (and (1 - p) / (1 - p + eps) of the gfocal derivative) loses bits when p is near 1, as
in the reference model's own fp32 formula.  Elements whose float64 sensitivity to p, times SIGMOID_ULPS ulps of 1, exceeds the relative
tolerance may move by that much more (grad_errors); they must be rare (SIGMOID_SHARE) and stay within SIGMOID_CAP, and every other
element is held to the plain 5e-5.  The top-1 hit count is exact except for bags whose float64 top-two margin is below TOP1_BOUND
(counted and printed).
"""
import numpy as np
import pytest
import torch

from tests.cpr_loss_ref import cpr_loss_ref, oracle_bag_logits, point_valid
from tests.helpers import scale_rel_err

pytestmark = pytest.mark.gpu

LB_MAXK = 320

GRAD_TOL = 5e-5
SIGMOID_ULPS = 8               # absolute error of the fp32 sigmoid near 1, in ulps of 1 (__expf + __fdividef: 4; doubled)
SIGMOID_SHARE = 1e-2           # at most this fraction of the gradient elements may need the sigmoid allowance (float64: <= 5.2e-3 here)
SIGMOID_CAP = 5e-3             # ... and there the plain scale-relative error stays below this (float64 allowance: <= 3.0e-2 here)
LOSS_TOL = 1e-5
TOP1_BOUND = 1e-5
EPS = 1e-6
PAD_VALUE = 50.0
H_MAP, W_MAP = 13, 21


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from pointtinybenchmark_b200 import ops as _ops
    return _ops


def ceil_to(n, m):
    return (n + m - 1) // m * m


def offset_table(K, stride, seed=0):
    """(K,2) fp32 CPU offset table with the centre LAST: K = 1 (centre only), a ring table (K = 4 r (r + 1) + 1), or 320 (the tile kernel's
    largest bag: the radius-8 rings, 31 extra points inside the radius and the centre)."""
    from pointtinybenchmark_b200 import ops as _ops
    if K == 1:
        return torch.zeros(1, 2)
    for r in range(1, 10):
        if 4 * r * (r + 1) + 1 == K:
            return _ops.circle_offsets(r, stride)
    assert K == LB_MAXK
    g = torch.Generator().manual_seed(seed)
    rings = _ops.circle_offsets(8, stride)[:-1]
    extra = (torch.rand(K - 1 - rings.shape[0], 2, generator=g) * 2 - 1) * (8 * stride)
    return torch.cat([rings, extra, torch.zeros(1, 2)]).float().contiguous()


def make_case(N, NP, K, stride, seed, n_per_img=(12, 0, 9), H=H_MAP, W=W_MAP):
    """seeded CPU inputs: logit map (pad columns = PAD_VALUE), bags with the edge cases listed in the module docstring, a neg mask."""
    g = torch.Generator().manual_seed(seed)
    B = len(n_per_img)
    LD = 2 * NP
    pad_hw = torch.tensor([[H * stride - (b * stride) // 2, W * stride - b * 3] for b in range(B)], dtype=torch.int32)
    cs, ls, bi = [], [], []
    for b, n in enumerate(n_per_img):
        if n == 0:
            continue
        ph, pw = float(pad_hw[b, 0]), float(pad_hw[b, 1])
        c = torch.rand(n, 2, generator=g) * torch.tensor([pw + 4 * stride, ph + 4 * stride]) - 2 * stride
        if n >= 6:
            c[0] = torch.tensor([0.0, 0.0])                          # centre exactly at the origin
            c[1] = torch.tensor([pw, ph])                            # at the pad edge: the centre sample is invalid
            c[2] = c[3]                                              # duplicated centre
            c[4] = torch.tensor([-1000.0, -1000.0])                  # far outside: every sample invalid, label weight 0
            c[5] = torch.tensor([pw + 1000.0, 3.0])
        cs.append(c)
        ls.append(torch.randint(0, N, (n,), generator=g))
        bi.append(torch.full((n,), b, dtype=torch.int32))
    centers = torch.cat(cs).float().contiguous()
    labels = torch.cat(ls).int()
    bag_img = torch.cat(bi)
    lens = list(n_per_img)
    img_ptr = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32)
    lmap = torch.full((B, H, W, LD), PAD_VALUE)
    lmap[..., :N] = torch.randn(B, H, W, N, generator=g) * 2.0 - 1.0
    lmap[..., NP:NP + N] = torch.randn(B, H, W, N, generator=g) * 2.0
    neg_mask = (torch.rand(B, H, W, N, generator=g) < 0.7).to(torch.uint8)
    off = offset_table(K, stride, seed)
    return dict(lmap=lmap.contiguous(), centers=centers, labels=labels, bag_img=bag_img, img_ptr=img_ptr, pad_hw=pad_hw,
                offsets=off, neg_mask=neg_mask, N=N, NP=NP, LD=LD, K=off.shape[0], stride=float(stride), B=B, H=H, W=W)


def to_dev(c):
    return {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in c.items()}


def scales(gt, neg, mil=True):
    s = dict(mil=0.37 if mil else 0.0, gt=0.29 if gt else 0.0, neg=0.011 if neg else 0.0)
    return s, {k: torch.tensor([v], device='cuda') for k, v in s.items()}


def check_forward(what, c, ref, bl,weight, bag_prob, loss, stats, mt, lw):
    """bit-exact sampled logits / validity, then the MIL forward outputs against the float64 reference; returns the error dict."""
    N, NP = c['N'], c['NP']
    o32 = oracle_bag_logits(c['lmap'], c['centers'], c['bag_img'], c['offsets'], c['stride'])
    blc = bl.cpu()
    assert torch.equal(blc[..., :N], o32[..., :N]) and torch.equal(blc[..., NP:NP + N], o32[..., NP:NP + N]), \
        f'{what}: sampled logits differ from the oracle fp32 grid_sample'
    assert torch.equal(weight.cpu().bool(), point_valid(c['centers'], c['bag_img'], c['offsets'], c['pad_hw'])), f'{what}: validity'
    assert torch.equal(lw.cpu().double(), ref['label_weight']), f'{what}: label weight'
    assert float(stats[0]) == ref['stats'][0], f'{what}: #bags with weight {float(stats[0])} != {ref["stats"][0]}'
    errs = dict(prob=scale_rel_err(bag_prob, ref['bag_prob']), loss=scale_rel_err(loss, ref['mil_sum'].reshape(1)))
    assert float((bag_prob.cpu().double() - ref['bag_prob']).abs().max()) <= TOP1_BOUND / 2, f'{what}: bag_prob off by > {TOP1_BOUND / 2}'
    mtc = mt.cpu()
    assert torch.equal(mtc[..., 0].double(), ref['mt_max']), f'{what}: max ins'
    assert torch.equal(mtc[..., 1] == 0, ref['inv_t'] == 0), f'{what}: clamp pattern of 1/T'
    errs['inv_t'] = scale_rel_err(mtc[..., 1], ref['inv_t'])
    close = ref['top_margin'] <= TOP1_BOUND
    hits_far = int(ref['hit'][~close].sum())
    hits_close_lo, hits_close_hi = hits_far, hits_far + int(close.sum())
    assert hits_close_lo <= float(stats[1]) <= hits_close_hi, f'{what}: top-1 hits {float(stats[1])} outside [{hits_close_lo}, {hits_close_hi}]'
    errs['top1_within_bound'] = int(close.sum())
    for k in ('prob', 'loss', 'inv_t'):
        assert errs[k] <= LOSS_TOL, f'{what}: {k} error {errs[k]:.2e} > {LOSS_TOL}'
    return errs


def gfocal_sums(ops, d, bl, weight, G, K, N, LD, M):
    wc = weight[:, K - 1].contiguous()
    gt = ops.gfocal_fwd(bl[:, K - 1], G, N, K * LD, d['labels'], wc, EPS)
    neg = ops.gfocal_fwd(d['lmap'], M, N, LD, None, d['neg_mask'], EPS)
    return wc, gt, neg


def check_grad(what, c, grad, ref, errs):
    N, NP, LD = c['N'], c['NP'], c['LD']
    g = grad.cpu()
    pad = torch.ones(LD, dtype=torch.bool)
    pad[:N] = False
    pad[NP:NP + N] = False
    assert bool((g[..., pad] == 0).all()), f'{what}: non-zero gradient in the pad columns'
    errs.update(grad_errors(g, ref['grad'], ref['kappa']))
    print(f'[cpr loss kernels] {what}: ' + ', '.join(f'{k} {v:.1e}' if isinstance(v, float) else f'{k} {v}' for k, v in errs.items()))
    assert_grad_errors(what, errs)


def grad_errors(a, b, kappa):
    """errors of a gradient a against the float64 reference b, with tests/helpers.scale_rel_err's floor max(|b|, rms(b)):
      grad          plain scale-relative error over all elements (printed);
      grad_plain    the same over the elements whose sigmoid allowance SIGMOID_ULPS * 2^-24 * kappa is below GRAD_TOL * floor / 4
                    (kappa = d gradient / d probability, tests/cpr_loss_ref.probability_sensitivity): held to GRAD_TOL;
      sigmoid_share fraction of elements above that line: held to SIGMOID_SHARE;
      grad_sigmoid  on those elements, |a - b| / (GRAD_TOL * floor + allowance) (held to 1) and the plain error (held to SIGMOID_CAP)."""
    a, b, kappa = a.detach().double().cpu(), b.detach().double().cpu(), kappa.detach().double().cpu()
    floor = torch.clamp(b.abs(), min=max(float(b.pow(2).mean().sqrt()), 1e-30))
    err = (a - b).abs()
    allowance = SIGMOID_ULPS * 2.0 ** -24 * kappa
    big = allowance > 0.25 * GRAD_TOL * floor
    rel = err / floor
    out = dict(grad=float(rel.max()), grad_plain=float(rel[~big].max()) if bool((~big).any()) else 0.0,
               sigmoid_share=float(big.double().mean()), grad_sigmoid=float(rel[big].max()) if bool(big.any()) else 0.0,
               grad_sigmoid_model=float((err / (GRAD_TOL * floor + allowance))[big].max()) if bool(big.any()) else 0.0)
    return out


def assert_grad_errors(what, e):
    assert e['grad_plain'] <= GRAD_TOL, f'{what}: gradient error {e["grad_plain"]:.2e} > {GRAD_TOL}'
    assert e['sigmoid_share'] <= SIGMOID_SHARE, f'{what}: {e["sigmoid_share"]:.2e} of the elements need the sigmoid allowance'
    assert e['grad_sigmoid_model'] <= 1.0 and e['grad_sigmoid'] <= SIGMOID_CAP, \
        f'{what}: gradient error {e["grad_sigmoid"]:.2e} where the fp32 sigmoid loses bits (model ratio {e["grad_sigmoid_model"]:.2f})'


def run_tiles(ops, c, gt=True, neg=True, what=''):
    d = to_dev(c)
    B, H, W, N, NP, LD, K = c['B'], c['H'], c['W'], c['N'], c['NP'], c['LD'], c['K']
    G, M = c['centers'].shape[0], B * H * W
    s, sd = scales(gt, neg)
    ref = cpr_loss_ref(c['lmap'], N, NP, c['centers'], c['bag_img'], c['offsets'], c['stride'], c['pad_hw'], c['labels'], EPS,
                       s['mil'], s['gt'], s['neg'], neg_mask=c['neg_mask'])
    bl, weight, bag_prob, loss, stats, mt, lw = ops.bag_mil_fwd(d['lmap'], N, NP, d['centers'], d['bag_img'], d['offsets'], c['stride'],
                                                                d['pad_hw'], d['labels'], EPS)
    errs = check_forward(what, c, ref, bl,weight, bag_prob, loss, stats, mt, lw)
    wc, gsum, nsum = gfocal_sums(ops, d, bl, weight, G, K, N, LD, M)
    errs['gt_sum'] = scale_rel_err(gsum, ref['gt_sum'].reshape(1))
    errs['neg_sum'] = scale_rel_err(nsum, ref['neg_sum'].reshape(1))
    assert errs['gt_sum'] <= LOSS_TOL and errs['neg_sum'] <= LOSS_TOL, f'{what}: gfocal sums {errs}'

    def bwd():
        return ops.cpr_loss_bwd_map(bl, weight, mt, bag_prob, lw, d['labels'], d['centers'], d['img_ptr'], d['offsets'], (B, H, W, LD), N, NP,
                                    c['stride'], ops.offsets_reach(c['offsets']), EPS, scale_mil=sd['mil'],
                                    scale_gt=sd['gt'] if gt else None, valid_center=wc if gt else None,
                                    logit_map=d['lmap'] if neg else None, neg_mask=d['neg_mask'] if neg else None,
                                    scale_neg=sd['neg'] if neg else None)
    g1 = bwd()
    g2 = bwd()
    assert torch.equal(g1, g2), f'{what}: the tile kernel gave different bits on two calls'
    check_grad(what, c, g1, ref, errs)


@pytest.mark.parametrize('K', [1, 9, 49, 289, 320])
@pytest.mark.parametrize('N', [1, 9, 16, 25, 33, 48, 64, 80])
def test_tile_kernel(ops, N, K):
    NP = ceil_to(N, 16)
    stride = 4 if (N + K) % 2 else 8
    c = make_case(N, NP, K, stride, seed=1000 * N + K)
    run_tiles(ops, c, what=f'tiles N={N} NP={NP} LD={2 * NP} K={c["K"]} stride={stride}')


@pytest.mark.parametrize('gt,neg', [(False, False), (True, False), (False, True)])
@pytest.mark.parametrize('N', [9, 80])
def test_tile_kernel_terms(ops, N, gt, neg):
    NP = ceil_to(N, 16)
    c = make_case(N, NP, 49, 8, seed=77 + N)
    run_tiles(ops, c, gt=gt, neg=neg, what=f'tiles N={N} LD={2 * NP} K=49 gt={gt} neg={neg}')


@pytest.mark.parametrize('N', [9, 80])
def test_tile_kernel_many_gts(ops, N):
    """one image with 1100 GTs on a 13 x 21 map: more than LB_MAXCAND (1024) candidate bags per tile, record-buffer flushes."""
    NP = ceil_to(N, 16)
    c = make_case(N, NP, 9, 4, seed=5 + N, n_per_img=(1100, 0, 7))
    run_tiles(ops, c, what=f'tiles N={N} LD={2 * NP} K=9 G={c["centers"].shape[0]}')


def run_scatter(ops, c, what, fused=True, gt=True, neg=True):
    d = to_dev(c)
    B, H, W, N, NP, LD, K = c['B'], c['H'], c['W'], c['N'], c['NP'], c['LD'], c['K']
    G, M = c['centers'].shape[0], B * H * W
    s, sd = scales(gt, neg)
    ref = cpr_loss_ref(c['lmap'], N, NP, c['centers'], c['bag_img'], c['offsets'], c['stride'], c['pad_hw'], c['labels'], EPS,
                       s['mil'], s['gt'], s['neg'], neg_mask=c['neg_mask'])
    if fused:
        bl, weight, bag_prob, loss, stats, mt, lw = ops.bag_mil_fwd(d['lmap'], N, NP, d['centers'], d['bag_img'], d['offsets'],
                                                                    c['stride'], d['pad_hw'], d['labels'], EPS)
    else:
        bl, _, valid = ops.bag_gather(d['lmap'], d['centers'], d['bag_img'], d['offsets'], c['stride'], d['pad_hw'], pts=False)
        weight = valid.float().contiguous()
        bag_prob, loss, stats, mt, lw = ops.mil_loss_fwd(bl, N, NP, weight, d['labels'], EPS, want_aux=True)
    errs = check_forward(what, c, ref, bl,weight, bag_prob, loss, stats, mt, lw)
    wc, gsum, nsum = gfocal_sums(ops, d, bl, weight, G, K, N, LD, M)
    errs['gt_sum'] = scale_rel_err(gsum, ref['gt_sum'].reshape(1))
    errs['neg_sum'] = scale_rel_err(nsum, ref['neg_sum'].reshape(1))
    assert errs['gt_sum'] <= LOSS_TOL and errs['neg_sum'] <= LOSS_TOL, f'{what}: gfocal sums {errs}'
    dl = torch.zeros((B, H, W, LD), device='cuda')
    if neg:
        ops.gfocal_bwd(d['lmap'], M, N, LD, None, d['neg_mask'], EPS, sd['neg'], dl, LD, accumulate=True)
    ops.cpr_loss_bwd_scatter(bl, weight, mt, bag_prob, lw, d['labels'], d['centers'], d['bag_img'], d['offsets'], dl, N, NP, c['stride'],
                             EPS, scale_mil=sd['mil'], scale_gt=sd['gt'] if gt else None, valid_center=wc if gt else None)
    check_grad(what, c, dl, ref, errs)


@pytest.mark.parametrize('K', [1, 49, 361])
@pytest.mark.parametrize('N', [1, 3, 8, 9, 33, 80, 100, 128])
def test_scatter_kernel(ops, N, K):
    NP = ceil_to(N, 8)
    stride = 8 if (N + K) % 2 else 4
    c = make_case(N, NP, K, stride, seed=2000 * N + K)
    run_scatter(ops, c, f'scatter N={N} NP={NP} K={c["K"]} stride={stride}')


@pytest.mark.parametrize('N', [129, 200, 256])
def test_scatter_kernel_wide(ops, N):
    """more classes than ptb_cpr_bag_mil_fwd takes: ptb_cpr_bag_gather + ptb_mil_loss_fwd(want_aux) feed the scatter kernel."""
    NP = ceil_to(N, 8)
    c = make_case(N, NP, 49, 4, seed=3000 + N)
    run_scatter(ops, c, f'scatter (gather + mil_loss_fwd) N={N} NP={NP} K=49', fused=False)


def test_scatter_kernel_many_gts(ops):
    c = make_case(9, 16, 9, 8, seed=11, n_per_img=(1100, 0, 7))
    run_scatter(ops, c, f'scatter N=9 K=9 G={c["centers"].shape[0]}')


@pytest.mark.parametrize('N,K,stride', [(13, 49, 4), (80, 289, 8)])
def test_staged_chain(ops, N, K, stride):
    """round-1 chain (grid-cell bags and PTB_LOSS_BWD=staged use it): mil_loss_bwd -> gfocal_bwd (centre) -> bag_gather_bwd -> gfocal_bwd (neg)."""
    NP = ceil_to(N, 8)
    c = make_case(N, NP, K, stride, seed=4000 + N)
    d = to_dev(c)
    B, H, W, LD, K = c['B'], c['H'], c['W'], c['LD'], c['K']
    G, M = c['centers'].shape[0], B * H * W
    s, sd = scales(True, True)
    ref = cpr_loss_ref(c['lmap'], N, NP, c['centers'], c['bag_img'], c['offsets'], c['stride'], c['pad_hw'], c['labels'], EPS,
                       s['mil'], s['gt'], s['neg'], neg_mask=c['neg_mask'])
    bl, _, valid = ops.bag_gather(d['lmap'], d['centers'], d['bag_img'], d['offsets'], c['stride'], d['pad_hw'], pts=False)
    weight = valid.float().contiguous()
    bag_prob, loss, stats, mt, lw = ops.mil_loss_fwd(bl, N, NP, weight, d['labels'], EPS, want_aux=True)
    what = f'staged N={N} K={K} stride={stride}'
    errs = check_forward(what, c, ref, bl,weight, bag_prob, loss, stats, mt, lw)
    wc = weight[:, K - 1].contiguous()
    dbl = torch.zeros_like(bl)
    ops.mil_loss_bwd(bl, N, NP, weight, d['labels'], EPS, bag_prob, sd['mil'], grad_out=dbl)
    ops.gfocal_bwd(bl[:, K - 1], G, N, K * LD, d['labels'], wc, EPS, sd['gt'], dbl[:, K - 1], K * LD, accumulate=True)
    dl = ops.bag_gather_bwd(dbl, (B, H, W, LD), d['centers'], d['bag_img'], d['offsets'], c['stride'])
    ops.gfocal_bwd(d['lmap'], M, N, LD, None, d['neg_mask'], EPS, sd['neg'], dl, LD, accumulate=True)
    check_grad(what, c, dl, ref, errs)


@pytest.mark.parametrize('N,extra', [(1, 3), (7, 1), (33, 15), (100, 4)])
@pytest.mark.parametrize('wmode', ['label_float', 'mask_uint8'])
def test_gfocal_kernels(ops, N, extra, wmode):
    """ptb_gfocal_sigmoid_fwd / _bwd on rows wider than the class count (row_stride = N + extra, grad row stride wider still), with a
    target label and a per-row float weight (gt term) or without a target and a per-element 0/1 mask (neg term); accumulate on and off."""
    g = torch.Generator().manual_seed(N * 10 + extra)
    M, rs, grs = 1537, N + extra, N + extra + 5
    x = torch.randn(M, rs, generator=g) * 3.0
    x[:, N:] = PAD_VALUE
    if wmode == 'label_float':
        tgt = torch.randint(0, N, (M,), generator=g).int()
        w = (torch.rand(M, generator=g) < 0.8).float() * torch.rand(M, generator=g)
        q = torch.zeros(M, N, dtype=torch.float64)
        q[torch.arange(M), tgt.long()] = 1.0
        w64 = w.double()[:, None]
    else:
        tgt = None
        w = (torch.rand(M, N, generator=g) < 0.6).to(torch.uint8)
        q = torch.zeros(M, N, dtype=torch.float64)
        w64 = w.double()
    from oracle import cpr as ocpr
    from tests.cpr_loss_ref import probability_sensitivity
    x64 = x[:, :N].double().requires_grad_(True)
    ref = ocpr.gfocal_loss(x64.sigmoid(), q, w64, EPS).sum()
    scale = 0.61
    (ref * scale).backward()
    kappa = probability_sensitivity(x64.detach(), q, w64, EPS, scale)
    xd, wd = x.cuda(), w.cuda()
    td = tgt.cuda() if tgt is not None else None
    s = ops.gfocal_fwd(xd, M, N, rs, td, wd, EPS)
    e_f = scale_rel_err(s, ref.detach().reshape(1))
    base = torch.randn(M, grs, generator=g)
    assert e_f <= LOSS_TOL, f'gfocal N={N}: sum error {e_f:.2e}'
    for acc in (False, True):
        gd = base.clone().cuda()
        ops.gfocal_bwd(xd, M, N, rs, td, wd, EPS, torch.tensor([scale], device='cuda'), gd, grs, accumulate=acc)
        gc = gd.cpu()
        assert torch.equal(gc[:, N:], base[:, N:]), 'columns past num_classes of the gradient rows must stay untouched'
        got = gc[:, :N].double() - (base[:, :N].double() if acc else 0.0)
        what = f'gfocal N={N} row_stride={rs} {wmode} accumulate={acc}'
        errs = grad_errors(got, x64.grad, kappa)
        print(f'[cpr loss kernels] {what}: sum {e_f:.1e}, ' + ', '.join(f'{k} {v:.1e}' for k, v in errs.items()))
        assert_grad_errors(what, errs)
