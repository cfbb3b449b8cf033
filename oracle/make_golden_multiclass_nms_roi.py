"""Runs the REAL reference multiclass_nms (core/post_processing/bbox_nms.py:7-94) on the RoI-head-shaped inputs of oracle/roi_nms.py
and writes tests/golden/multiclass_nms_roi.npz.  (test infrastructure)

Run in the build container only (needs /root/reference):   python -m oracle.make_golden_multiclass_nms_roi
The unmodified reference is imported through oracle/_mmcv_stub.py, whose batched_nms restates mmcv's (class offset, the split_thr
branch).  The stub's single-class NMS defers to torchvision when it is installed; here it is oracle.p2p.nms, the same greedy
IoU > thr rule with ties visited lower index first.  Every case is ASSERTED equal to oracle.p2p.multiclass_nms before it is stored.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import p2p as op2p, roi_nms  # noqa: E402
from oracle import _mmcv_stub  # noqa: E402
from oracle.make_golden import GOLD, eq  # noqa: E402


def stub_nms(boxes, scores, iou_threshold, offset=0, score_threshold=0, max_num=-1):
    assert offset == 0
    keep = op2p.nms(boxes, scores, iou_threshold)
    if max_num > 0:
        keep = keep[:max_num]
    return torch.cat([boxes[keep], scores[keep, None]], 1), keep


def main():
    try:
        import torchvision  # noqa: F401
    except ImportError:
        _mmcv_stub.nms = stub_nms                       # batched_nms looks `nms` up in the stub module at call time
    _mmcv_stub.install()
    from mmdet.core.post_processing.bbox_nms import multiclass_nms as ref_mnms
    out = {}
    for name, c in roi_nms.CASES.items():
        b, s, f = roi_nms.inputs(name)
        bt, st = torch.from_numpy(b), torch.from_numpy(s)
        ft = torch.from_numpy(f) if f is not None else None
        cfg = dict(type='nms', iou_threshold=roi_nms.IOU)
        rd, rl, rk = ref_mnms(bt, st, roi_nms.SCORE_THR, dict(cfg), c['max_num'], score_factors=ft, return_inds=True)
        od, ol, ok, inds = op2p.multiclass_nms(bt, st, roi_nms.SCORE_THR, roi_nms.IOU, c['max_num'], nms_cfg=cfg, score_factors=ft)
        eq(od, rd, f'{name} dets'); eq(ol, rl, f'{name} labels'); eq(ok, rk, f'{name} keep')
        out[f'{name}_dets'], out[f'{name}_labels'], out[f'{name}_keep'] = rd.numpy(), rl.numpy(), rk.numpy()
        out[f'{name}_cand_count'] = np.int64(len(inds))
        out[f'{name}_checksum'] = np.array([roi_nms.checksum(b), roi_nms.checksum(s), roi_nms.checksum(f if f is not None else 0)])
        print(f'[golden] {name}: {len(inds)} candidates, {len(rk)} kept (max_num {c["max_num"]})')
    path = os.path.join(GOLD, 'multiclass_nms_roi.npz')
    np.savez_compressed(path, **out)
    print(f'[golden] {path}: {os.path.getsize(path) / 1024:.0f} KiB')


if __name__ == '__main__':
    main()
