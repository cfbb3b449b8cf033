"""CPU: the RoI head's multiclass_nms call (1000 RoIs x 80 classes + background, class-specific boxes (n, 320), score_thr 0.05,
IoU 0.5) recorded from the REAL reference function in tests/golden/multiclass_nms_roi.npz (oracle/make_golden_multiclass_nms_roi.py),
against the oracle restatement and against the host restatement of the class-specific kernels (tests/nms_cls_ref.py).  The GPU run
of the same cases is tests/test_gpu_multiclass_nms_roi.py."""
import os

import numpy as np
import pytest
import torch

from oracle import p2p as op2p, roi_nms
from tests import nms_cls_ref as cref, nms_ref as ref


@pytest.fixture(scope='module')
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, 'multiclass_nms_roi.npz'))


@pytest.mark.parametrize('name', list(roi_nms.CASES))
def test_inputs_are_the_recorded_ones(gold, name):
    b, s, f = roi_nms.inputs(name)
    got = [roi_nms.checksum(b), roi_nms.checksum(s), roi_nms.checksum(f if f is not None else 0)]
    assert np.array_equal(np.array(got), gold[f'{name}_checksum']), name


@pytest.mark.parametrize('name', list(roi_nms.CASES))
def test_oracle_matches_the_reference_golden(gold, name):
    c = roi_nms.CASES[name]
    b, s, f = roi_nms.inputs(name)
    cfg = dict(type='nms', iou_threshold=roi_nms.IOU)
    d, l, k, inds = op2p.multiclass_nms(torch.from_numpy(b), torch.from_numpy(s), roi_nms.SCORE_THR, roi_nms.IOU, c['max_num'],
                                        nms_cfg=cfg, score_factors=None if f is None else torch.from_numpy(f))
    assert len(inds) == int(gold[f'{name}_cand_count'])
    assert np.array_equal(k.numpy(), gold[f'{name}_keep'])
    assert np.array_equal(l.numpy(), gold[f'{name}_labels'])
    assert np.array_equal(d.numpy(), gold[f'{name}_dets'])


def restated(name):
    c = roi_nms.CASES[name]
    b, s, f = roi_nms.inputs(name)
    ks, thr = cref.glue_scores(s, roi_nms.SCORE_THR, f)
    mk = 1024 if c['max_num'] <= 0 else c['max_num']
    return cref.image(b.reshape(roi_nms.N, roi_nms.C, 4), ks, thr, roi_nms.IOU, mk), b, ks, thr


@pytest.mark.parametrize('name', list(roi_nms.CASES))
def test_restatement_matches_the_reference_golden(gold, name):
    r, _, _, _ = restated(name)
    assert r['cand_count'] == int(gold[f'{name}_cand_count'])
    assert np.array_equal(r['keep'], gold[f'{name}_keep'])
    assert np.array_equal(r['labels'], gold[f'{name}_labels'])
    assert np.array_equal(r['det'], gold[f'{name}_dets'])


def test_the_cases_reach_both_branches_and_the_slow_path():
    seen = {}
    for name in roi_nms.CASES:
        r, b, ks, thr = restated(name)
        p = cref.expected_path(b.reshape(roi_nms.N, roi_nms.C, 4), ks, thr)
        seen[name] = (p['path'], p['split'])
    assert seen['below'] == ('class', False) and seen['factors'] == ('class', False) and seen['sparse'] == ('class', False)
    assert seen['above'] == ('class', True) and seen['clustered'] == ('class', True)
    assert seen['slow'] == ('global', False)
    r, b, ks, thr = restated('slow')
    split = cref.image(b.reshape(roi_nms.N, roi_nms.C, 4), ks, thr, roi_nms.IOU, 100, branch='split')
    assert r['branch'] == 'offset' and not np.array_equal(r['flat'], split['flat']), 'the slow case must separate the two branches'


SOFT_CASES = [(m, opt) for m in ('linear', 'gaussian', 'naive') for opt in ('cls_boxes', 'factors', 'agnostic')]


def soft_inputs(seed, n=120, C=7):
    """class-specific boxes (n, 4C) around n objects, scores (n, C+1), factors (n,): a few hundred candidates."""
    rng = np.random.default_rng(seed)
    ctr = rng.random((n, 2)) * 200
    wh = rng.random((n, 2)) * 30 + 10
    base = np.concatenate([ctr - wh / 2, ctr + wh / 2], 1)
    boxes = (base[:, None] + rng.normal(0, 3.0, (n, C, 4))).astype(np.float32)
    boxes = np.concatenate([np.minimum(boxes[..., :2], boxes[..., 2:]), np.maximum(boxes[..., :2], boxes[..., 2:])], -1)
    scores = (rng.random((n, C + 1)) ** 2).astype(np.float32)
    return boxes.reshape(n, 4 * C).astype(np.float32), scores, rng.random(n).astype(np.float32)


def soft_expected(method, opt, seed):
    """the oracle's soft-NMS (oracle.p2p.multiclass_nms with type='soft_nms') and the host restatement of the kernels on one case."""
    b, s, f = soft_inputs(seed)
    n, C = s.shape[0], s.shape[1] - 1
    cfg = dict(type='soft_nms', iou_threshold=0.3, sigma=0.5, min_score=1e-3, method=method)
    if opt == 'agnostic':
        cfg['class_agnostic'] = True
    sf = f if opt == 'factors' else None
    od, ol, ok, _ = op2p.multiclass_nms(torch.from_numpy(b), torch.from_numpy(s), 0.05, 0.3, 100, nms_cfg=cfg,
                                        score_factors=None if sf is None else torch.from_numpy(sf))
    ks, thr = cref.glue_scores(s, 0.05, sf)
    soft = dict(sigma=0.5, min_score=1e-3, method=method)
    if opt == 'agnostic':                                    # one class: the (box, class) pairs flattened
        r = ref.image(b.reshape(n * C, 4), ks.reshape(n * C, 1), thr, 0.3, 100, soft_cfg=soft)
        r['labels'] = ref.candidates(ks, thr)[r['keep']] % C
    else:
        r = cref.image(b.reshape(n, C, 4), ks, thr, 0.3, 100, soft_cfg=soft)
    return (od.numpy(), ol.numpy(), ok.numpy()), r, (b, s, f)


@pytest.mark.parametrize('method,opt', SOFT_CASES, ids=[f'{m}-{o}' for m, o in SOFT_CASES])
def test_soft_nms_restatement_matches_the_oracle(method, opt):
    """the restatement of the class-specific / score_factors / class_agnostic soft-NMS against oracle.p2p's mmcv restatement:
    keep, labels and boxes exact, decayed scores within 4 ulp per decay, over the rows the gaussian method decides."""
    (od, ol, ok), r, _ = soft_expected(method, opt, seed=300 + SOFT_CASES.index((method, opt)))
    assert r['count'] == len(ok) and r['count'] > 20
    e = r['exact_upto']
    assert np.array_equal(r['keep'][:e], ok[:e]) and np.array_equal(r['labels'][:e], ol[:e])
    assert np.array_equal(r['det'][:e, :4], od[:e, :4])
    tol = 4 * 2.0 ** -23 * (np.arange(e) + 1) * np.abs(od[:e, 4].astype(np.float64))
    assert (np.abs(r['det'][:e, 4].astype(np.float64) - od[:e, 4]) <= tol).all()
