"""CPU: oracle/tile_test.py against the real reference's TwoStageDetector.tile_aug_test and StandardRoIHead.aug_test
(tests/golden/tile_test_*.npz, written by oracle/make_golden_tile_test.py): every case's detections, per class, in order."""
import os

import numpy as np
import pytest
import torch

from oracle import tile_test as ott

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def _compare(d, l, f, C):
    d, l = d.numpy(), l.numpy()
    for k in range(C):
        a, b = d[l == k], f['dets'][f['labels'] == k]
        assert a.shape == b.shape, f'class {k}: oracle {a.shape[0]} rows, reference {b.shape[0]}'
        np.testing.assert_allclose(a, b, rtol=0, atol=1e-5)
    assert [int((l == k).sum()) for k in range(C)] == f['counts'].tolist()


@pytest.mark.parametrize('name', [n for n, c in ott.CASES.items() if not c['direct']])
def test_oracle_tile_aug_test_against_reference(name):
    f = np.load(os.path.join(GOLD, f'tile_test_{name}.npz'))
    c, inp = ott.CASES[name], ott.case_inputs(name)
    props = [torch.from_numpy(p) for p in np.split(f['rpn_props'], np.cumsum(f['rpn_counts'])[:-1])]
    stats = {}
    d, l = ott.tile_aug_test(inp['feats'], [m[0] for m in inp['img_metas']], props, inp['roi_weights'], ott.roi_head_spec(name), c['rpn'],
                             c['rcnn'], stats=stats)
    _compare(d, l, f, c['C'])
    assert stats['merge_rows'] == int(f['merge_rows'])
    if name == 'tinyperson12':
        assert stats['merge_rows'] >= 10000                  # mmcv batched_nms's class-by-class branch at the cross-tile merge
    if name == 'empty':
        assert len(f['dets']) == 0


def test_oracle_aug_test_against_reference():
    name = 'direct'
    f = np.load(os.path.join(GOLD, f'tile_test_{name}.npz'))
    c, inp = ott.CASES[name], ott.case_inputs(name)
    d, l = ott.aug_test(inp['feats'], [m[0] for m in inp['img_metas']], inp['proposals'], inp['roi_weights'], ott.roi_head_spec(name), c['rcnn'])
    _compare(d, l, f, c['C'])
    assert int(f['mismatch_raises']) == 1
