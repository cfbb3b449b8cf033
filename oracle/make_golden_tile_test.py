"""Pins oracle/tile_test.py against the REAL reference and writes tests/golden/tile_test_*.npz.  (test infrastructure)

Run in the build container only (needs /root/reference):   python -m oracle.make_golden_tile_test
The unmodified reference mmdet package is imported through oracle/_mmcv_stub.py (mmcv.ops.RoIAlign bound to oracle.roi_head.RoIAlign).
For every case of oracle.tile_test.CASES a reference RPNHead and StandardRoIHead are built with the case's seeded weights, and
TwoStageDetector.tile_aug_test runs with a stand-in `self` whose extract_feats returns the case's per-aug features (the direct case calls
StandardRoIHead.aug_test on seeded proposals instead, once with offsets every aug keeps, once with an offset that drops proposals of one
aug, where the reference raises).  The oracle runs on the RPN's per-aug proposals and its detections are ASSERTED equal (count per class,
rows within 1e-5).  Stored: the reference RPN's per-aug proposals, the number of rows at the cross-tile merge, the reference's detections and labels (class-major, as bbox2result splits them) and their per-class counts;
the inputs are regenerated from the seeds."""
import copy
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import roi_head as orh  # noqa: E402
from oracle import tile_test as ott  # noqa: E402
from oracle import _mmcv_stub as stub  # noqa: E402
from oracle.make_golden import GOLD  # noqa: E402


def cfgdict(d):
    return stub.CfgDict({k: cfgdict(v) if isinstance(v, dict) else v for k, v in d.items()})


def build(HEADS, name):
    c = ott.CASES[name]
    inp = ott.case_inputs(name)
    rk, hk = ott.head_kwargs(name)
    rpn = HEADS.build(dict(type='RPNHead', **rk, test_cfg=cfgdict(c['rpn'])))
    rpn.load_state_dict(inp['rpn_weights'], strict=True)
    roi = HEADS.build(dict(type='StandardRoIHead', **hk, test_cfg=cfgdict(c['rcnn'])))
    roi.bbox_head.load_state_dict(inp['roi_weights'], strict=True)
    return c, inp, rpn.eval(), roi.eval()


def flat(bbox_results):
    d = np.concatenate(bbox_results, 0).astype(np.float32)
    lab = np.concatenate([np.full(len(r), k, np.int64) for k, r in enumerate(bbox_results)])
    return d, lab, np.array([len(r) for r in bbox_results], np.int64)


def check(name, d, lab, od, ol):
    ol = ol.numpy()
    od = od.numpy()
    for k in range(int(max(lab.max(initial=-1), ol.max(initial=-1)) + 1)):
        a, b = d[lab == k], od[ol == k]
        assert a.shape == b.shape, f'{name} class {k}: reference {a.shape[0]} rows, oracle {b.shape[0]}'
        assert np.allclose(a, b, rtol=0, atol=1e-5), f'{name} class {k}: max diff {np.abs(a - b).max()}'


def golden_case(HEADS, name):
    from mmdet.models.detectors.two_stage import TwoStageDetector
    c, inp, rpn, roi = build(HEADS, name)
    out = dict(seed=np.int64(c['seed']))
    with torch.no_grad():
        if c['direct']:
            feats = inp['feats']
            res = roi.aug_test(feats, [inp['proposals'].clone()], copy.deepcopy(inp['img_metas']))[0]
            d, lab, cnt = flat(res)
            od, ol = ott.aug_test([[x for x in f] for f in feats], [m[0] for m in inp['img_metas']], inp['proposals'], inp['roi_weights'],
                                  ott.roi_head_spec(name), c['rcnn'])
            check(name, d, lab, od, ol)
            bad = copy.deepcopy(inp['img_metas'])
            bad[1][0]['tile_offset'] = (110, 90)
            try:
                roi.aug_test(feats, [inp['proposals'].clone()], bad)
                raise AssertionError(f'{name}: the reference accepted proposal sets of different sizes')
            except RuntimeError:
                out['mismatch_raises'] = np.int64(1)
        else:
            metas = copy.deepcopy(inp['img_metas'])
            props = [rpn.simple_test_rpn(f, m)[0] for f, m in zip(inp['feats'], metas)]
            fake = type('Detector', (), {})()
            fake.extract_feats = lambda imgs: inp['feats']
            fake.rpn_head, fake.roi_head = rpn, roi
            fake.test_cfg = cfgdict(dict(rpn=c['rpn'], rcnn=c['rcnn']))
            res = TwoStageDetector.tile_aug_test(fake, None, metas, rescale=False)[0]
            assert all('tile_offset' not in m[0] for m in metas)
            d, lab, cnt = flat(res)
            od, ol = ott.tile_aug_test([[x for x in f] for f in inp['feats']], [m[0] for m in inp['img_metas']], props, inp['roi_weights'],
                                       ott.roi_head_spec(name), c['rpn'], c['rcnn'])
            check(name, d, lab, od, ol)
            out['rpn_counts'] = np.array([len(p) for p in props], np.int64)
            out['rpn_props'] = torch.cat(props).numpy()          # the reference RPN's per-aug proposals: the oracle's CPU input
            stats = {}
            ott.tile_aug_test([[x for x in f] for f in inp['feats']], [m[0] for m in inp['img_metas']], props, inp['roi_weights'],
                              ott.roi_head_spec(name), c['rpn'], c['rcnn'], stats=stats)
            out['merge_rows'] = np.int64(stats['merge_rows'])
    out.update(dets=d, labels=lab, counts=cnt)
    path = os.path.join(GOLD, f'tile_test_{name}.npz')
    np.savez_compressed(path, **out)
    print(f'[golden] {path}: {len(d)} detections, per class {cnt.tolist()}, merge rows {out.get("merge_rows")}')


def main():
    torch.set_num_threads(1)
    stub.KNOWN['mmcv.ops']['RoIAlign'] = orh.RoIAlign
    stub.Registry.__contains__ = lambda self, key: self.get(key) is not None
    HEADS = stub.load_reference()
    # mmcv.ops.nms is a function in mmcv; the stub also installs the mmcv.ops.nms module, which shadows it under `from mmcv.ops import nms`
    import mmdet.core.post_processing.merge_augs as merge_augs
    merge_augs.nms = stub.nms
    for name in (sys.argv[1:] or ott.CASES):
        golden_case(HEADS, name)


if __name__ == '__main__':
    main()
