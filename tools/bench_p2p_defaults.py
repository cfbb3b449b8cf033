"""P2PHead at the reference class's own defaults (p2p_head.py:25-45: 4 point anchors per cell -> 320-channel cls_out,
CrossEntropyLoss(use_sigmoid=True) + MSELoss) at the BASELINE.json configs[2] shape: 16 images of 256 x 100 x 168 at stride 8 =
16 800 cells x 4 anchors = 67 200 proposals per image.  Prints one JSON line:
  p2p_defaults_infer_ms   P2PHead.simple_test per 16 images (towers + wgmma output convs + decode / top-k / NMS)
  p2p_defaults_train_ms   with --train: forward_train + backward per 16 images, 20 GT points per image, HungarianAssignerV2 topk_k 5.
                          At 67 200 rows the matching is past the cluster kernel's 17 600-column limit and runs its one-CTA
                          global-memory path (lsap.cu).
  p2p_softmax_infer_ms    with --softmax: the same head with CrossEntropyLoss(use_sigmoid=False): 4 anchors x 81 outputs (80 classes +
                          background) = 324-channel cls_out, softmax decode / top-k
  p2p_softmax_train_ms    with --softmax --train: its training step (softmax cross-entropy kernel)
CUDA events, L2 flushed (256 MB write) before every timed call, mean over the timed calls.  Writes nothing.

    python tools/bench_p2p_defaults.py [--train] [--softmax] [--iters N]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pointtinybenchmark_b200 import p2p_head  # noqa: E402,F401  (registers the head)
from pointtinybenchmark_b200.registry import build_head  # noqa: E402

B, C, H, W, STRIDE, NCLS = 16, 256, 100, 168, 8, 80
PAD_HW, IMG_HW = (800, 1344), (800, 1333)
TRAIN_CFG = dict(neg_weight=1.0, assigner=dict(type='HungarianAssignerV2', cls_costs=dict(type='FocalLossCost', weight=2.0),
                                               reg_costs=dict(type='DisCostV2', weight=0.1, norm_with_img_wh=False), topk_k=5),
                 sampler=dict(type='PseudoSampler'))
TEST_CFG = dict(nms_pre=1000, min_bbox_size=0, score_thr=0.05, pseudo_wh=(32, 32), nms=dict(type='nms', iou_threshold=0.5),
                max_per_img=100)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--train', action='store_true', help='also time the training step')
    ap.add_argument('--softmax', action='store_true', help='also time the head with softmax classification (4 anchors x 81 outputs)')
    ap.add_argument('--iters', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device (there is no CPU fallback)')
    dev = torch.device('cuda:0')
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)

    def ktime(fn, n):
        for _ in range(3):
            fn()
        ts = []
        for _ in range(n):
            flush.add_(1.0)
            s, e = torch.cuda.Event(True), torch.cuda.Event(True)
            s.record(); fn(); e.record(); torch.cuda.synchronize()
            ts.append(s.elapsed_time(e))
        return float(np.mean(ts))

    cfg = dict(type='P2PHead', norm_cfg=dict(type='GN', num_groups=32, requires_grad=True), num_classes=NCLS, in_channels=C,
               feat_channels=C, stacked_convs=4, strides=[STRIDE], test_cfg=TEST_CFG)
    x = torch.randn(B, C, H, W, generator=torch.Generator().manual_seed(11)).to(dev).contiguous(memory_format=torch.channels_last)
    metas = [dict(pad_shape=PAD_HW + (3,), img_shape=IMG_HW + (3,), scale_factor=[1.0, 1.0, 1.0, 1.0])] * B
    out = dict(workload=f'P2PHead reference defaults (4 anchors / cell, cls_out {4 * NCLS} ch), {B} x ({C}x{H}x{W}), '
                        f'{H * W * 4} proposals per image, random-init weights',
               device=torch.cuda.get_device_name(dev))
    g = torch.Generator().manual_seed(13)
    gtb = []
    for _ in range(B):
        cxy = torch.rand(20, 2, generator=g) * torch.tensor([1300., 780.]) + 10
        gtb.append(torch.cat([cxy - 8, cxy + 8], 1).to(dev))
    gtl = [torch.randint(0, NCLS, (20,), generator=g).to(dev) for _ in range(B)]

    def run(prefix, hcfg):
        head = build_head(hcfg).to(dev).eval()
        with torch.no_grad():
            out[f'{prefix}_infer_ms'] = ktime(lambda: head.simple_test((x,), metas), args.iters)
        out['tower_backend'] = head.last_tower_backend
        del head
        if args.train:
            head = build_head(dict(hcfg, train_cfg=TRAIN_CFG)).to(dev).train()
            xt = x.clone().requires_grad_(True)

            def step():
                head.zero_grad(set_to_none=True)
                ls = head.forward_train((xt,), metas, gtb, gtl)
                (sum(ls['loss_cls']) + sum(ls['loss_pts'])).backward()
            out[f'{prefix}_train_ms'] = ktime(step, max(1, args.iters // 2 + 1))

    run('p2p_defaults', cfg)
    if args.softmax:
        run('p2p_softmax', dict(cfg, loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0)))
    print(json.dumps(out))


if __name__ == '__main__':
    main()
