"""GPU: ptb_p2p_cost_matrix_terms, HungarianAssignerV2's cost lists (FocalLossCost, ClassificationCostV2 sigmoid / softmax, ZeroCost,
DisCostV2 p=1 / p=2) in one kernel — every term against ATen's fp32 CPU result and a float64 restatement, the summation order, the
golden vectors of the real reference (tests/golden/p2p_match_costs.npz) and P2PHead.loss with the paper's costs.

Tolerances against ATen's CPU result, as measured on an H100 host: ZeroCost and DisCostV2(p=1) bit for bit;
ClassificationCostV2(use_sigmoid=True) within 1 ulp (1 element of 625 differed); FocalLossCost 1e-6 scale-relative (logf against
ATen's vectorised log: up to 512 ulps where pos - neg cancels); ClassificationCostV2(use_sigmoid=False) within SOFTMAX_ULPS (the
kernel divides by the row sum, ATen multiplies by its reciprocal and sums in another order; measured at most 3 ulps);
DisCostV2(p=2) within 1 ulp on the direct path (measured 0) and within the matmul formulation's own rounding on the other (ATen's
result there depends on the host's BLAS: up to 16 ulps measured where |x|^2 + |y|^2 - 2 x.y cancels).  The summation order is
checked bit for bit against the fp32 sum, in the reference's order, of the kernel's own single-term costs."""
import os

import numpy as np
import pytest
import torch

from oracle import p2p as op2p, p2p_match_costs as omc, p2p_softmax as osm
from tests.helpers import assert_close

pytestmark = pytest.mark.gpu

SOFTMAX_ULPS = 4
FOCAL = dict(kind='FocalLossCost', weight=2.0, alpha=0.25, gamma=2, eps=1e-12)
TERMS = {
    'focal': FOCAL,
    'focal_a3': dict(kind='FocalLossCost', weight=-0.5, alpha=0.3, gamma=2, eps=1e-12),
    'sigmoid': dict(kind='ClassificationCostV2_sigmoid', weight=1.5),
    'softmax': dict(kind='ClassificationCostV2_softmax', weight=2.0),
    'zero': dict(kind='ZeroCost', weight=0.0),
}
SHAPES = [(25, 25), (26, 1), (1, 26), (200, 12)]
IMG = (110, 117, 3)


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from pointtinybenchmark_b200 import ops
    return ops


def ulps(a, b):
    """elementwise distance in units in the last place of two fp32 arrays (+0 and -0 are 0 apart)"""
    def key(x):
        i = np.ascontiguousarray(np.asarray(x, np.float32)).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7fffffff), i)
    return np.abs(key(a) - key(b))


def inputs(seed, N, n, C1, spread=2.0):
    """Q = 2N + 3 proposals, N of them selected by row_idx; points in a (Q, 3) buffer (ldp 3)"""
    g = torch.Generator().manual_seed(seed)
    h, w = IMG[:2]
    Q = 2 * N + 3
    cls = torch.randn(Q, C1, generator=g) * spread
    pts3 = torch.rand(Q, 3, generator=g) * torch.tensor([w, h, 1.0])
    gts = torch.rand(n, 2, generator=g) * torch.tensor([w, h])
    labels = torch.randint(0, min(C1, 80), (n,), generator=g)
    ridx = torch.randperm(Q, generator=g)[:N]
    return cls, pts3, gts, labels, ridx


def run(ops, cls, pts3, gts, labels, ridx, terms):
    dev = torch.device('cuda:0')
    p = pts3.to(dev)
    return ops.p2p_cost_matrix_terms(cls.to(dev), p[:, :2], ridx.int().to(dev), gts.to(dev), labels.int().to(dev), terms,
                                     float(IMG[1]), float(IMG[0])).cpu()


def oracle(cls, pts3, gts, labels, ridx, terms):
    """the reference's sum; a list of ZeroCost alone sums to the integer 0"""
    return torch.zeros(len(ridx), len(gts)) + omc.cost_matrix(pts3[ridx, :2].contiguous(), cls[ridx], gts, labels, IMG, terms)


def float64_term(t, cls, pts, gts, labels):
    """float64 restatement of one term from its formula (match_cost.py), independent of ATen's fp32 kernels"""
    x = cls.double()[:, labels]
    w = float(np.float32(t['weight']))
    k = t['kind']
    if k == 'FocalLossCost':
        p = torch.sigmoid(x)
        neg = -(1 - p + t['eps']).log() * (1 - t['alpha']) * p.pow(t['gamma'])
        pos = -(p + t['eps']).log() * t['alpha'] * (1 - p).pow(t['gamma'])
        return (pos - neg) * w
    if k == 'ClassificationCostV2_sigmoid':
        return -torch.sigmoid(x) * w
    if k == 'ClassificationCostV2_softmax':
        return -cls.double().softmax(-1)[:, labels] * w
    if k == 'ZeroCost':
        return torch.zeros(x.shape, dtype=torch.float64)
    f = torch.tensor([IMG[1], IMG[0]], dtype=torch.float64) if t['norm_with_img_wh'] else 1.0
    return torch.cdist(pts.double() / f, gts.double() / f, p=t['p']) * w


def check_term(got, ref32, ref64, bound, what):
    """got within `bound` of ATen's fp32 result: an ulp count (0: bit for bit), or 'rel' for 1e-6 scale-relative, or an array of
    absolute bounds; and 1e-4 scale-relative of float64"""
    u = ulps(got.numpy(), ref32.numpy())
    print(f'[{what}] max {u.max()} ulps from ATen, {int((u > 0).sum())} / {u.size} elements differ')
    if isinstance(bound, str):
        assert_close(got, ref32, 1e-6, f'{what} vs ATen')
    elif isinstance(bound, int):
        assert u.max() <= bound, f'{what}: {u.max()} ulps from ATen (bound {bound}), {int((u > 0).sum())} elements differ'
    else:
        err = (got.double() - ref32.double()).abs()
        assert bool((err <= bound).all()), f'{what}: {int((err > bound).sum())} elements beyond the bound'
    assert_close(got, ref64, 1e-4, f'{what} vs float64')


def mm_bound(pts, gts, t):
    """|error| of ATen's fp32 cdist matmul formulation: a few ulps of |x|^2 + |y|^2 in d^2, i.e. of (|x|^2 + |y|^2) / 2d in d, plus
    the sqrt's and the weight's rounding"""
    f = torch.tensor([IMG[1], IMG[0]], dtype=torch.float64) if t['norm_with_img_wh'] else 1.0
    x, y = pts.double() / f, gts.double() / f
    s = (x * x).sum(1)[:, None] + (y * y).sum(1)[None, :]
    d = torch.cdist(x, y)
    eps = 2.0 ** -23
    return t['weight'] * (4 * eps * s / (2 * d).clamp(min=1e-30) + 4 * eps * d)


@pytest.mark.parametrize('shape', SHAPES, ids=lambda s: f'{s[0]}x{s[1]}')
@pytest.mark.parametrize('C1', [80, 81])
@pytest.mark.parametrize('name', list(TERMS))
def test_classification_term(ops, name, C1, shape):
    """each classification term alone, at the C columns of a sigmoid head and the C + 1 of a softmax head"""
    N, n = shape
    t = TERMS[name]
    cls, pts3, gts, labels, ridx = inputs(11 + N + n + C1, N, n, C1)
    got = run(ops, cls, pts3, gts, labels, ridx, [t])
    ref64 = float64_term(t, cls[ridx], pts3[ridx, :2], gts, labels)
    bound = dict(softmax=SOFTMAX_ULPS, sigmoid=1, zero=0).get(name, 'rel')
    check_term(got, oracle(cls, pts3, gts, labels, ridx, [t]), ref64, bound, f'{name} C1={C1} {N}x{n}')


@pytest.mark.parametrize('shape', SHAPES, ids=lambda s: f'{s[0]}x{s[1]}')
@pytest.mark.parametrize('norm', [True, False])
@pytest.mark.parametrize('p', [1, 2])
def test_distance_term(ops, p, norm, shape):
    """DisCostV2 alone on both sides of torch.cdist's 25-row dispatch, with and without the division by (w, h)"""
    N, n = shape
    t = dict(kind='DisCostV2', weight=5e-2 if p == 2 else 0.1, p=p, norm_with_img_wh=norm)
    cls, pts3, gts, labels, ridx = inputs(23 + N + n + p, N, n, 80)
    got = run(ops, cls, pts3, gts, labels, ridx, [t])
    ref64 = float64_term(t, cls[ridx], pts3[ridx, :2], gts, labels)
    bound = 0 if p == 1 else (mm_bound(pts3[ridx, :2], gts, t) if max(N, n) > 25 else 1)
    check_term(got, oracle(cls, pts3, gts, labels, ridx, [t]), ref64, bound, f'p{p} norm={norm} {N}x{n}')


def test_weight_zero_terms_are_exact(ops):
    terms = [dict(TERMS['softmax'], weight=0.0), dict(TERMS['sigmoid'], weight=0.0), dict(FOCAL, weight=0.0),
             dict(kind='DisCostV2', weight=0.0, p=2, norm_with_img_wh=True), dict(kind='DisCostV2', weight=0.0, p=1, norm_with_img_wh=False)]
    cls, pts3, gts, labels, ridx = inputs(5, 60, 9, 81)
    got, ref = run(ops, cls, pts3, gts, labels, ridx, terms), oracle(cls, pts3, gts, labels, ridx, terms)
    assert np.array_equal(got.numpy().view(np.int32), ref.numpy().view(np.int32))


@pytest.mark.parametrize('shape', [(0, 5), (7, 0), (0, 0)])
def test_empty_rows_or_gts(ops, shape):
    N, n = shape
    cls, pts3, gts, labels, ridx = inputs(3, max(N, 1), n, 81)
    ridx = ridx[:N]
    got = run(ops, cls, pts3, gts, labels, ridx, [TERMS['softmax'], dict(kind='DisCostV2', weight=5e-2, p=2, norm_with_img_wh=True)])
    assert tuple(got.shape) == (N, n)


def test_summation_order_is_the_references(ops):
    """sum(cls_costs) + sum(reg_costs) from 0, in list order: bit for bit against the fp32 sum of the kernel's single-term costs"""
    ct = [FOCAL, TERMS['sigmoid'], TERMS['zero'], TERMS['softmax'], TERMS['focal_a3'], dict(TERMS['sigmoid'], weight=3.0)]
    rt = [dict(kind='DisCostV2', weight=0.1, p=1, norm_with_img_wh=True), dict(kind='DisCostV2', weight=5e-2, p=2, norm_with_img_wh=True),
          dict(kind='DisCostV2', weight=0.3, p=1, norm_with_img_wh=False)]
    for N, n in ((200, 12), (20, 5)):
        cls, pts3, gts, labels, ridx = inputs(7 + N, N, n, 81)
        got = run(ops, cls, pts3, gts, labels, ridx, ct + rt)
        cs, rs = torch.zeros(N, n), torch.zeros(N, n)
        for t in ct:
            cs = cs + run(ops, cls, pts3, gts, labels, ridx, [t])
        for t in rt:
            rs = rs + run(ops, cls, pts3, gts, labels, ridx, [t])
        assert np.array_equal(got.numpy().view(np.int32), (cs + rs).numpy().view(np.int32)), (N, n)
        assert_close(got, oracle(cls, pts3, gts, labels, ridx, ct + rt), 1e-6, 'nine terms vs the oracle')


def test_eight_terms_per_list(ops):
    """the longest lists: 8 classification terms (every kind) and 8 DisCostV2 terms, against the oracle's sum"""
    ct = [FOCAL, TERMS['sigmoid'], TERMS['softmax'], TERMS['zero'], TERMS['focal_a3'], dict(TERMS['softmax'], weight=0.5),
          dict(TERMS['sigmoid'], weight=-1.0), TERMS['zero']]
    rt = [dict(kind='DisCostV2', weight=0.01 * (i + 1), p=1 + i % 2, norm_with_img_wh=i % 3 == 0) for i in range(8)]
    cls, pts3, gts, labels, ridx = inputs(8, 100, 10, 81)
    got, ref = run(ops, cls, pts3, gts, labels, ridx, ct + rt), oracle(cls, pts3, gts, labels, ridx, ct + rt)
    assert_close(got, ref, 1e-6, 'sixteen terms')
    with pytest.raises(RuntimeError, match='at most 8'):
        run(ops, cls, pts3, gts, labels, ridx, ct + [FOCAL] + rt)
    with pytest.raises(RuntimeError, match='at most 8'):
        run(ops, cls, pts3, gts, labels, ridx, ct + rt + rt[:1])


# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, 'p2p_match_costs.npz'))


def exact_kinds(terms):
    return all(t['kind'] in ('FocalLossCost', 'ClassificationCostV2_sigmoid', 'ZeroCost') or t.get('p') == 1 for t in terms)


@pytest.mark.parametrize('name', list(omc.CASES))
def test_golden_cost_and_assignments(ops, gold, name):
    from pointtinybenchmark_b200 import assigners
    dev = torch.device('cuda:0')
    terms, N, n, _ = omc.CASES[name]
    t = {k: torch.from_numpy(gold[f'{name}_{k}']).to(dev) for k in ('pts', 'cls', 'gts', 'labels')}
    cost = ops.p2p_cost_matrix_terms(t['cls'], t['pts'], None, t['gts'], t['labels'].int(), terms, float(omc.IMG_SHAPE[1]),
                                     float(omc.IMG_SHAPE[0])).cpu().numpy()
    ref = gold[f'{name}_cost']
    if exact_kinds(terms):
        assert np.array_equal(cost.view(np.int32), ref.view(np.int32)), f'{name}: cost not bit-identical to the reference'
    else:
        err = np.abs(cost.astype(np.float64) - ref)
        print(f'[{name}] max |cost - reference| {err.max():.3e}, {int((cost != ref).sum())} / {cost.size} differ')
        assert err.max() <= 2e-6 * max(1.0, float(np.abs(ref).max())), name
    cc, rc = omc.cost_config(terms)
    for k in (1, 5):
        want = gold[f'{name}_gt_inds_k{k}']
        out = torch.zeros(N, dtype=torch.int64, device=dev)
        st = ops.hungarian_v2_batch(torch.from_numpy(ref).to(dev).view(-1), [(N, n)], k, out, [0])
        assert int(st[0]) == 0 and np.array_equal(out.cpu().numpy().astype(np.int32), want), f'{name}: matching of the golden cost, topk {k}'
        r = assigners.HungarianAssignerV2(cls_costs=cc, reg_costs=rc, topk_k=k).assign(t['pts'], t['cls'], t['gts'], t['labels'],
                                                                                        dict(img_shape=omc.IMG_SHAPE))
        assert np.array_equal(r.gt_inds.cpu().numpy().astype(np.int32), want), f'{name}: kernel cost + matching, topk {k}'


PAPER_TRAIN_CFG = dict(neg_weight=1.0, assigner=dict(type='HungarianAssignerV2', cls_costs=dict(type='ClassificationCostV2',
                                                                                                use_sigmoid=False, weight=2.0),
                                                     reg_costs=dict(type='DisCostV2', weight=5e-2, p=2), topk_k=5),
                       sampler=dict(type='PseudoSampler'))


@pytest.fixture(scope='module')
def head_case(ops, gold):
    from pointtinybenchmark_b200 import p2p_head  # noqa: F401  (registers the head)
    from pointtinybenchmark_b200.registry import build_head
    inp = osm.inputs(int(gold['head_seed']))
    d = inp['cfgd']
    cfg = osm.softmax_cfg(use_sigmoid=False, num_classes=d['num_classes'], stride=d['stride'])
    with torch.no_grad():
        oc, op_ = op2p.head_forward(inp['x'], inp['weights'], cfg)
    head = build_head(dict(type='P2PHead', num_classes=d['num_classes'], in_channels=d['C'], feat_channels=d['C'], stacked_convs=4,
                           strides=[d['stride']], point_anchor=d['point_anchor'], norm_cfg=dict(type='GN', num_groups=32, requires_grad=True),
                           loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0), train_cfg=PAPER_TRAIN_CFG)).cuda()
    return head, inp, oc, op_


def test_head_loss_with_the_paper_costs(ops, gold, head_case):
    """P2PHead(softmax CrossEntropyLoss) with ClassificationCostV2(use_sigmoid=False) + DisCostV2(p=2): assignments exact, losses 1e-4
    and gradients 2e-4 against the real reference head"""
    head, inp, oc, op_ = head_case
    dev = torch.device('cuda:0')
    assert [t['kind'] for t in head.assign['terms']] == ['ClassificationCostV2_softmax', 'DisCostV2']
    co, po = oc.to(dev).requires_grad_(True), op_.to(dev).requires_grad_(True)
    got = head.loss([co], [po], [b.to(dev) for b in inp['gt_bboxes']], [l.to(dev) for l in inp['gt_labels']], inp['img_metas'])
    (sum(got['loss_cls']) + sum(got['loss_pts'])).backward()
    assert np.array_equal(head._last_assign['gt_inds'].cpu().numpy().astype(np.int32), gold['head_gt_inds']), 'assignments'
    assert np.array_equal(torch.stack(head._last_targets['labels']).cpu().numpy(), gold['head_labels']), 'labels'
    for k in ('loss_cls', 'loss_pts'):
        assert_close(torch.stack(got[k]).detach(), torch.from_numpy(gold['head_' + k]), 1e-4, k)
    assert_close(co.grad.flatten()[::37], torch.from_numpy(gold['head_grad_cls_sub']), 2e-4, 'd/d cls_out')
    assert_close(po.grad.flatten(), torch.from_numpy(gold['head_grad_pts_sub']), 2e-4, 'd/d pts_out')


@pytest.mark.parametrize('bad', [float('nan'), float('inf')], ids=['nan', 'inf'])
def test_nonfinite_logit_under_the_softmax_cost_raises(ops, head_case, bad):
    from pointtinybenchmark_b200 import assigners
    dev = torch.device('cuda:0')
    cls, pts3, gts, labels, _ = inputs(2, 40, 6, 81)
    cls[7, 3] = bad
    A = assigners.HungarianAssignerV2(cls_costs=dict(type='ClassificationCostV2', weight=2.0),
                                      reg_costs=dict(type='DisCostV2', weight=5e-2, p=2), topk_k=1)
    with pytest.raises(ValueError, match='invalid numeric entries'):
        A.assign(pts3[:, :2].contiguous().to(dev), cls.to(dev), gts.to(dev), labels.to(dev), dict(img_shape=IMG))
    head, inp, oc, op_ = head_case
    oc = oc.clone()
    oc[1, 5, 3, 4] = bad                     # a valid cell of image 1
    with pytest.raises(ValueError, match='invalid numeric entries'):
        head.loss([oc.to(dev)], [op_.to(dev)], [b.to(dev) for b in inp['gt_bboxes']], [l.to(dev) for l in inp['gt_labels']],
                  inp['img_metas'])
