"""GPU: multiclass_nms with class-specific boxes, the RoI head's call, and soft-NMS with every option, on the kernels of csrc/nms.cu.

  golden    post_processing.multiclass_nms(bboxes (1000, 320), scores (1000, 81), 0.05, IoU 0.5, max_num 100 / -1) with and without
            score_factors: dets, labels and keep bit-equal to the REAL reference (tests/golden/multiclass_nms_roi.npz) and to the host
            restatement (tests/nms_cls_ref.py), which also fixes the path each case takes: the offset branch below 10000 candidates,
            the split branch above, and the exact global path on the `slow` image whose two branches differ
  soft      soft-NMS (linear, gaussian, naive) with class-specific boxes, score_factors and class_agnostic against oracle.p2p's
            restatement of mmcv's soft_nms and against the host restatement; linear at the RoI head's size on all three paths
  limits    P = 4096 boxes accepted and 4097 refused by both class-specific entry points; gaussian refuses an image on its
            candidates' own zero-area boxes only
"""
import os
import re

import numpy as np
import pytest
import torch

from oracle import roi_nms
from tests import nms_cls_ref as cref
from tests.test_multiclass_nms_roi_golden import SOFT_CASES, restated, soft_expected

F32 = np.float32


@pytest.fixture(scope='module')
def pp():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from pointtinybenchmark_b200 import post_processing
    return post_processing


def _np(t):
    return t.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(roi_nms.CASES))
def test_roi_head_call_matches_the_reference_golden(pp, golden_dir, name):
    z = np.load(os.path.join(golden_dir, 'multiclass_nms_roi.npz'))
    c = roi_nms.CASES[name]
    b, s, f = roi_nms.inputs(name)
    dev = torch.device('cuda:0')
    args = (torch.from_numpy(b).to(dev), torch.from_numpy(s).to(dev), roi_nms.SCORE_THR, dict(type='nms', iou_threshold=roi_nms.IOU),
            c['max_num'])
    sf = None if f is None else torch.from_numpy(f).to(dev)
    d, l, k = pp.multiclass_nms(*args, score_factors=sf, return_inds=True)
    assert np.array_equal(_np(k), z[f'{name}_keep']), name
    assert np.array_equal(_np(l), z[f'{name}_labels']), name
    assert np.array_equal(_np(d), z[f'{name}_dets']), name
    r, bb, ks, thr = restated(name)
    assert np.array_equal(_np(k), r['keep']) and np.array_equal(_np(d), r['det'])
    path = cref.expected_path(bb.reshape(roi_nms.N, roi_nms.C, 4), ks, thr)
    want = dict(slow=('global', False), above=('class', True), clustered=('class', True)).get(name, ('class', False))
    assert (path['path'], path['split']) == want, name
    d2, l2 = pp.multiclass_nms(*args, score_factors=sf)
    assert torch.equal(d2, d) and torch.equal(l2, l), 'two calls differ'


@pytest.mark.gpu
def test_roi_head_call_counts_every_candidate(pp):
    """the op level: cand_count and count per image of a batch of the three path cases, against the restatement."""
    from pointtinybenchmark_b200 import ops
    names = ('below', 'above', 'slow')
    bs, ss, rs = [], [], []
    for name in names:
        r, b, ks, thr = restated(name)
        bs.append(b.reshape(roi_nms.N, roi_nms.C, 4)); ss.append(ks); rs.append(r)
    cnt, det, lab, keep, cc = ops.multiclass_nms_boxes(torch.from_numpy(np.stack(bs)).cuda(), torch.from_numpy(np.stack(ss)).cuda(),
                                                       roi_nms.SCORE_THR, roi_nms.IOU, 100)
    for i, r in enumerate(rs):
        assert int(cc[i]) == r['cand_count'] and int(cnt[i]) == r['count'], names[i]
        assert np.array_equal(_np(keep[i, :r['count']]), r['keep']) and np.array_equal(_np(lab[i, :r['count']]), r['labels'])
        assert np.array_equal(_np(det[i, :r['count']]), r['det'])


def _check_soft(d, l, k, r, od, ol, ok, method, what):
    n = len(_np(k))
    if r['all_exact']:
        assert n == r['count'], what
    e = min(r['exact_upto'], n)
    d, l, k = _np(d), _np(l), _np(k)
    for want_k, want_l, want_d in ((r['keep'], r['labels'], r['det']), (ok, ol, od)):
        assert np.array_equal(k[:e], want_k[:e]) and np.array_equal(l[:e], want_l[:e]), what
        assert np.array_equal(d[:e, :4], want_d[:e, :4]), what
    if method == 'gaussian':                   # row k has been decayed at most k times: 4 ulp per expf and product
        for want in (r['det'], od):
            tol = 4 * 2.0 ** -23 * (np.arange(e) + 1) * np.abs(want[:e, 4].astype(np.float64))
            assert (np.abs(d[:e, 4].astype(np.float64) - want[:e, 4]) <= tol).all(), what
    else:
        assert np.array_equal(d[:, 4], r['det'][:, 4]), what
        assert np.array_equal(d[:, 4], od[:, 4]), what


@pytest.mark.gpu
@pytest.mark.parametrize('method,opt', SOFT_CASES, ids=[f'{m}-{o}' for m, o in SOFT_CASES])
def test_soft_nms_options_match_the_oracle_and_the_restatement(pp, method, opt):
    (od, ol, ok), r, (b, s, f) = soft_expected(method, opt, seed=300 + SOFT_CASES.index((method, opt)))
    cfg = dict(type='soft_nms', iou_threshold=0.3, sigma=0.5, min_score=1e-3, method=method)
    if opt == 'agnostic':
        cfg['class_agnostic'] = True
    sf = torch.from_numpy(f).cuda() if opt == 'factors' else None
    d, l, k = pp.multiclass_nms(torch.from_numpy(b).cuda(), torch.from_numpy(s).cuda(), 0.05, cfg, 100, score_factors=sf, return_inds=True)
    _check_soft(d, l, k, r, od, ol, ok, method, f'{method}-{opt}')


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['below', 'above', 'slow', 'factors'])
def test_soft_nms_linear_at_roi_head_size(pp, name):
    """linear soft-NMS on the 1000 x 80 cases: the per-class kernels with the merge (offset and split branch) and the global kernel."""
    b, s, f = roi_nms.inputs(name)
    ks, thr = cref.glue_scores(s, roi_nms.SCORE_THR, f)
    soft = dict(sigma=0.5, min_score=1e-3, method='linear')
    r = cref.image(b.reshape(roi_nms.N, roi_nms.C, 4), ks, thr, roi_nms.IOU, 100, soft_cfg=soft)
    cfg = dict(type='soft_nms', iou_threshold=roi_nms.IOU, **soft)
    sf = None if f is None else torch.from_numpy(f).cuda()
    d, l, k = pp.multiclass_nms(torch.from_numpy(b).cuda(), torch.from_numpy(s).cuda(), roi_nms.SCORE_THR, cfg, 100, score_factors=sf,
                                return_inds=True)
    assert len(k) == r['count'] == 100
    assert np.array_equal(_np(k), r['keep']) and np.array_equal(_np(l), r['labels']) and np.array_equal(_np(d), r['det'])


@pytest.mark.gpu
def test_class_specific_entry_points_take_4096_boxes_and_refuse_4097(pp):
    from pointtinybenchmark_b200 import ops
    rng = np.random.default_rng(4096)
    C = 3
    ctr = rng.random((4097, 1, 2)) * 3000
    bx = np.concatenate([ctr - 8, ctr + 8], -1) + rng.normal(0, 1.0, (4097, C, 4))
    sc = (rng.random((4097, C)) * (rng.random((4097, C)) < 0.5)).astype(F32)
    bx = bx.astype(F32)
    for P in (4096, 4097):
        bt, st = torch.from_numpy(bx[None, :P]).cuda().contiguous(), torch.from_numpy(sc[None, :P]).cuda().contiguous()
        if P == 4097:
            with pytest.raises(RuntimeError, match='4096'):
                ops.multiclass_nms_boxes(bt, st, 0.05, 0.5, 100)
            with pytest.raises(RuntimeError, match='4096'):
                ops.multiclass_soft_nms(bt, st, None, 0.05, 0.5, 100)
            continue
        r = cref.image(bx[:P], sc[:P], 0.05, 0.5, 1024)
        cnt, det, lab, keep, cc = ops.multiclass_nms_boxes(bt, st, 0.05, 0.5, 1024)
        assert int(cc[0]) == r['cand_count'] and int(cnt[0]) == r['count']
        assert np.array_equal(_np(keep[0, :r['count']]), r['keep']) and np.array_equal(_np(det[0, :r['count']]), r['det'])
        soft = dict(sigma=0.5, min_score=1e-3, method='linear')
        r = cref.image(bx[:P], sc[:P], 0.05, 0.5, 1024, soft_cfg=soft)
        cnt, det, lab, keep, cc = ops.multiclass_soft_nms(bt, st, None, 0.05, 0.5, 1024, **soft)
        assert int(cnt[0]) == r['count']
        assert np.array_equal(_np(keep[0, :r['count']]), r['keep']) and np.array_equal(_np(det[0, :r['count']]), r['det'])


@pytest.mark.gpu
def test_gaussian_refusal_looks_at_each_candidates_own_box(pp):
    """two zero-area boxes refuse the image only when both belong to candidates: a (box, class) pair below score_thr does not count."""
    from pointtinybenchmark_b200 import ops
    rng = np.random.default_rng(77)
    P, C = 64, 4
    ctr = rng.random((P, 1, 2)) * 300
    bx = (np.concatenate([ctr - 10, ctr + 10], -1) + rng.normal(0, 1.0, (P, C, 4))).astype(F32)
    sc = (0.1 + 0.8 * rng.random((P, C))).astype(F32)
    bx[5, 2, 2] = bx[5, 2, 0]                           # zero-area boxes of (5, 2) and (9, 1)
    bx[9, 1, 3] = bx[9, 1, 1]
    soft = dict(sigma=0.5, min_score=1e-3, method='gaussian')
    both = torch.from_numpy(bx[None]).cuda()
    with pytest.raises(RuntimeError, match=re.escape('refused image(s) [0]')):
        ops.multiclass_soft_nms(both, torch.from_numpy(sc[None]).cuda(), None, 0.05, 0.3, 100, **soft)
    sc[9, 1] = 0.01                                     # (9, 1) is no candidate: one zero-area candidate box is accepted
    r = cref.image(bx, sc, 0.05, 0.3, 100, soft_cfg=soft)
    assert not r['refused']
    cnt, det, lab, keep, cc = ops.multiclass_soft_nms(both, torch.from_numpy(sc[None]).cuda(), None, 0.05, 0.3, 100, **soft)
    e = min(r['exact_upto'], int(cnt[0]))
    assert e > 10 and np.array_equal(_np(keep[0, :e]), r['keep'][:e]) and np.array_equal(_np(det[0, :e, :4]), r['det'][:e, :4])
