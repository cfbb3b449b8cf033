"""The RoI head's multiclass_nms on the GPU: B = 8 images x 1000 RoIs x 80 classes + background, class-specific boxes (1000, 320),
score_thr 0.05, IoU 0.5, max_per_img 100, the seeded inputs of oracle/roi_nms.py (images alternate between about 8 000 candidates,
mmcv's offset branch, and about 16 000, the split branch).  Times, with CUDA events, over --rounds alternating rounds of --iters calls:
  hard_per_image   post_processing.multiclass_nms(type='nms') once per image, as the head's get_bboxes calls it
  soft_per_image   the same with type='soft_nms', method 'linear'
  hard_batched     one ops.multiclass_nms_boxes call on the (8, 1000, 80, 4) batch
  soft_batched     one ops.multiclass_soft_nms call on it (linear)
and reports per batch of 8 images the median and the min-max over rounds.  The oracle (oracle.p2p.multiclass_nms, torch / numpy on
the host) runs once per kind on one image of each branch beside it.  Prints the card's name and power limit, then one JSON line.
Writes nothing.

    python tools/bench_multiclass_nms.py [--rounds 5] [--iters 10] [--warmup 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import p2p as op2p, roi_nms  # noqa: E402
from pointtinybenchmark_b200 import ops, post_processing  # noqa: E402

B = 8
IMAGES = ('below', 'above') * (B // 2)
HARD = dict(type='nms', iou_threshold=roi_nms.IOU)
SOFT = dict(type='soft_nms', iou_threshold=roi_nms.IOU, sigma=0.5, min_score=1e-3, method='linear')


def card():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0) + ', power limit unknown'


def timed(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_multiclass_nms: no CUDA device')
    print('card:', card(), flush=True)
    dev = torch.device('cuda:0')
    host = [roi_nms.inputs(n)[:2] for n in IMAGES]
    imgs = [(torch.from_numpy(b).to(dev), torch.from_numpy(s).to(dev)) for b, s in host]
    bb = torch.stack([b.view(roi_nms.N, roi_nms.C, 4) for b, _ in imgs]).contiguous()
    ss = torch.stack([s[:, :-1] for _, s in imgs]).contiguous()

    def per_image(cfg):
        return lambda: [post_processing.multiclass_nms(b, s, roi_nms.SCORE_THR, cfg, 100) for b, s in imgs]

    runs = {
        'hard_per_image': per_image(HARD),
        'soft_per_image': per_image(SOFT),
        'hard_batched': lambda: ops.multiclass_nms_boxes(bb, ss, roi_nms.SCORE_THR, roi_nms.IOU, 100),
        'soft_batched': lambda: ops.multiclass_soft_nms(bb, ss, None, roi_nms.SCORE_THR, roi_nms.IOU, 100, method='linear'),
    }
    for fn in runs.values():
        for _ in range(args.warmup):
            fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in runs}
    for _ in range(args.rounds):
        for k, fn in runs.items():
            ms[k].append(timed(fn, args.iters))
    out = dict(card=card(), images=B, rois=roi_nms.N, classes=roi_nms.C, rounds=args.rounds, iters=args.iters)
    for k, v in ms.items():
        out[k + '_ms'] = dict(median=round(statistics.median(v), 3), min=round(min(v), 3), max=round(max(v), 3))
        print(f'{k:16s} {statistics.median(v):8.3f} ms per batch of {B}  (min {min(v):.3f}, max {max(v):.3f})', flush=True)
    for kind, cfg in (('hard', HARD), ('soft', SOFT)):
        for name in ('below', 'above'):
            b, s = (torch.from_numpy(a) for a in roi_nms.inputs(name)[:2])
            t0 = time.perf_counter()
            op2p.multiclass_nms(b, s, roi_nms.SCORE_THR, roi_nms.IOU, 100, nms_cfg=cfg)
            dt = (time.perf_counter() - t0) * 1e3
            out[f'oracle_{kind}_{name}_ms_per_image'] = round(dt, 1)
            print(f'oracle {kind} {name}: {dt:.1f} ms per image (host)', flush=True)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
