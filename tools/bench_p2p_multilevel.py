"""P2PHead over five FPN levels against the single-level head, at the reference class's own defaults (4 point anchors per cell,
CrossEntropyLoss(use_sigmoid=True) + MSELoss, 80 classes): 16 images of 1333 x 800 (padded to 1344 x 800).

  multilevel    strides [8, 16, 32, 64, 128]: maps 100x168, 50x84, 25x42, 13x21, 7x11 of 256 channels, 89 600 proposals per image,
                5 chunks of 17 920 for the top-k, 5 x nms_pre = 5000 NMS points (the 8192-point NMS entry points)
  single        strides [8]: the 100x168 map alone, 67 200 proposals per image
For each: simple_test (towers + output convs + decode / top-k / NMS under torch.no_grad) and the training step (forward_train with
20 GT points per image + backward).  CUDA events around each call (which ends in a device synchronise), --iters timed calls after
--warmup, median and min-max in ms, and the peak memory of the timed calls.  The numbers are whatever this run measured; the card's
name, power limit and SM clocks are printed with them.  Prints one JSON line.  Writes nothing.

    python tools/bench_p2p_multilevel.py [--iters 20] [--warmup 3]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pointtinybenchmark_b200 import p2p_head  # noqa: E402,F401  (registers the head)
from pointtinybenchmark_b200.registry import build_head  # noqa: E402
from tools.bench_p2p_many_classes import TEST_CFG, TRAIN_CFG, card, timed  # noqa: E402

B, C, N_GT, NUM_CLASSES = 16, 256, 20, 80
PAD_HW, IMG_HW = (800, 1344), (800, 1333)
STRIDES = [8, 16, 32, 64, 128]


def map_hw(s):
    return -(-PAD_HW[0] // s), -(-PAD_HW[1] // s)


def run(strides, iters, warmup, dev):
    g = torch.Generator().manual_seed(len(strides))
    xs = [torch.relu(torch.randn(B, C, *map_hw(s), generator=g)).to(dev) for s in strides]
    metas = [dict(pad_shape=PAD_HW + (3,), img_shape=IMG_HW + (3,), scale_factor=[1.0] * 4) for _ in range(B)]
    gtb, gtl = [], []
    for _ in range(B):
        p = torch.rand(N_GT, 2, generator=g) * torch.tensor([IMG_HW[1], IMG_HW[0]])
        gtb.append(torch.cat([p - 8, p + 8], 1).to(dev))
        gtl.append(torch.randint(0, NUM_CLASSES, (N_GT,), generator=g).to(dev))
    head = build_head(dict(type='P2PHead', norm_cfg=dict(type='GN', num_groups=32, requires_grad=True), num_classes=NUM_CLASSES,
                           in_channels=C, feat_channels=C, stacked_convs=4, strides=strides, train_cfg=TRAIN_CFG,
                           test_cfg=TEST_CFG)).to(dev)
    out = dict(strides=strides, maps=[list(map_hw(s)) for s in strides],
               proposals_per_image=sum(h * w for h, w in map(map_hw, strides)) * head.num_points)
    head.eval()

    def infer():
        with torch.no_grad():
            head.simple_test(xs, metas)
    out['simple_test'] = timed(infer, iters, warmup)
    head.train()

    def step():
        head.zero_grad(set_to_none=True)
        ls = head.forward_train(xs, metas, gtb, gtl)
        (sum(ls['loss_cls']) + sum(ls['loss_pts'])).backward()
    out['train'] = timed(step, iters, warmup)
    del head
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_p2p_multilevel needs a CUDA device')
    dev = torch.device('cuda:0')
    torch.backends.cudnn.allow_tf32 = False
    res = dict(card=card(), batch=B, image=list(IMG_HW), num_classes=NUM_CLASSES,
               multilevel=run(STRIDES, args.iters, args.warmup, dev), single=run([8], args.iters, args.warmup, dev))
    print(f"card: {res['card']}  (measured numbers of this run)")
    for k in ('multilevel', 'single'):
        r = res[k]
        print(f"{k:10s} strides {r['strides']}: simple_test {r['simple_test']['ms_median']} ms "
              f"[{r['simple_test']['ms_min']}-{r['simple_test']['ms_max']}], train {r['train']['ms_median']} ms "
              f"[{r['train']['ms_min']}-{r['train']['ms_max']}], peak {r['train']['peak_gb']} GB")
    print(json.dumps(res))


if __name__ == '__main__':
    main()
