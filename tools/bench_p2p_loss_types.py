"""P2PHead's training step with each loss pair, in one process, the arms alternating step by step:

  focal_sl1      FocalLoss + SmoothL1Loss(beta 1/9)            (the shipped configs)
  ghmc_ghmr      GHMC(bins 30, momentum 0.75) + GHMR(mu 0.02)
  focal_l1       FocalLoss + L1Loss
  focal_bl1      FocalLoss + BalancedL1Loss (alpha 0.5, gamma 1.5, beta 1)
at two shapes:
  tinyperson     16 x 640 x 640 images, stride 4 (one 160 x 160 map), 1 class, 1 anchor (the shipped TinyPersonV2 setup)
  defaults       16 x 800 x 1333 images, stride 8 (one 100 x 168 map), 80 classes, 4 anchors (the reference class's defaults)
The training step is forward_train with 20 GT points per image + backward, timed with CUDA events (it ends in a device synchronise):
median and min-max of --iters steps per arm after --warmup.  The GHM histogram + weight step alone (ops.ghmc_bin_weights on the
step's (B, Q, C) logits, ops.ghmr_bin_weights on its points) is timed the same way over --iters launches.  The numbers are whatever
this run measured; the card's name, power limit and SM clocks are printed with them.  Prints one JSON line.  Writes nothing.

    python tools/bench_p2p_loss_types.py [--iters 20] [--warmup 3]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pointtinybenchmark_b200 import ops, p2p_head  # noqa: E402,F401  (registers the head)
from pointtinybenchmark_b200.registry import build_head  # noqa: E402
from tools.bench_p2p_many_classes import TRAIN_CFG, card, event_ms, summary  # noqa: E402

B, C, N_GT = 16, 256, 20
SHAPES = {
    'tinyperson': dict(pad=(640, 640), img=(640, 640), stride=4, num_classes=1, anchors=[(0., 0.)], pts_gamma=1.0, reg_norm=1.0),
    'defaults': dict(pad=(800, 1344), img=(800, 1333), stride=8, num_classes=80,
                     anchors=[(-0.25, -0.25), (0.25, -0.25), (0.25, 0.25), (-0.25, 0.25)], pts_gamma=100. / 8, reg_norm=1. / 8),
}
FOCAL = dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0)
ARMS = {
    'focal_sl1': (FOCAL, dict(type='SmoothL1Loss', beta=1.0 / 9.0, loss_weight=0.5)),
    'ghmc_ghmr': (dict(type='GHMC', bins=30, momentum=0.75, use_sigmoid=True, loss_weight=1.0),
                  dict(type='GHMR', mu=0.02, bins=10, momentum=0.7, loss_weight=1.0)),
    'focal_l1': (FOCAL, dict(type='L1Loss', loss_weight=0.5)),
    'focal_bl1': (FOCAL, dict(type='BalancedL1Loss', loss_weight=0.5)),
}


def run_shape(sh, iters, warmup, dev):
    s = sh['stride']
    H, W = -(-sh['pad'][0] // s), -(-sh['pad'][1] // s)
    g = torch.Generator().manual_seed(H * W)
    xs = [torch.relu(torch.randn(B, C, H, W, generator=g)).to(dev)]
    metas = [dict(pad_shape=sh['pad'] + (3,), img_shape=sh['img'] + (3,), scale_factor=[1.0] * 4) for _ in range(B)]
    gtb, gtl = [], []
    for _ in range(B):
        p = torch.rand(N_GT, 2, generator=g) * torch.tensor([sh['img'][1], sh['img'][0]])
        gtb.append(torch.cat([p - 8, p + 8], 1).to(dev))
        gtl.append(torch.randint(0, sh['num_classes'], (N_GT,), generator=g).to(dev))
    heads = {}
    for arm, (lc, lr) in ARMS.items():
        heads[arm] = build_head(dict(type='P2PHead', norm_cfg=dict(type='GN', num_groups=32, requires_grad=True),
                                     num_classes=sh['num_classes'], in_channels=C, feat_channels=C, stacked_convs=4, strides=[s],
                                     point_anchor=sh['anchors'], pts_gamma=sh['pts_gamma'], reg_norm=sh['reg_norm'],
                                     loss_cls=lc, loss_reg=lr, train_cfg=TRAIN_CFG)).to(dev).train()
    sd = heads['focal_sl1'].state_dict()          # the same weights in every arm
    for h in heads.values():
        h.load_state_dict(sd, strict=False)

    def step(h):
        h.zero_grad(set_to_none=True)
        ls = h.forward_train(xs, metas, gtb, gtl)
        (sum(ls['loss_cls']) + sum(ls['loss_pts'])).backward()

    for _ in range(warmup):
        for h in heads.values():
            step(h)
    torch.cuda.synchronize()
    ts = {arm: [] for arm in heads}
    for _ in range(iters):
        for arm, h in heads.items():
            ts[arm].append(event_ms(lambda: step(h)))
    out = dict(map=[H, W], proposals_per_image=H * W * len(sh['anchors']), train={a: summary(t) for a, t in ts.items()})
    # the GHM histogram + weight step alone, on the GHM arm's own last-step logits and targets
    h = heads['ghmc_ghmr']
    with torch.no_grad():
        outs = h(xs)
        _, pred, _, cls = h.get_pred_points(outs[0][0], outs[1][0], metas)
    tg = h._last_targets
    x, lab, lw = cls.contiguous(), torch.stack(tg['labels']), torch.stack(tg['label_weights'])
    p, gp, pw = pred.contiguous(), torch.stack(tg['gt_pts']), torch.stack(tg['pts_weights'])
    inv = h.row_inv_norm([(H, W)], dev)
    m, r = h.loss_cls, h.loss_reg
    for _ in range(warmup):
        ops.ghmc_bin_weights(x, lab, lw, m.edges, m.momentum, m.acc_sum)
    out['ghmc_bin_weights'] = summary([event_ms(lambda: ops.ghmc_bin_weights(x, lab, lw, m.edges, m.momentum, m.acc_sum))
                                       for _ in range(iters)])
    out['ghmc_logits_mb'] = round(x.numel() * 4 / 1e6, 1)
    out['ghmr_bin_weights'] = summary([event_ms(lambda: ops.ghmr_bin_weights(p, gp, pw, inv, 0.02, r.edges, r.momentum, r.acc_sum))
                                       for _ in range(iters)])
    del heads
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_p2p_loss_types needs a CUDA device')
    dev = torch.device('cuda:0')
    torch.backends.cudnn.allow_tf32 = False
    res = dict(card=card(), batch=B, arms={a: [lc['type'], lr['type']] for a, (lc, lr) in ARMS.items()},
               shapes={k: run_shape(sh, args.iters, args.warmup, dev) for k, sh in SHAPES.items()})
    print(f"card: {res['card']}  (measured numbers of this run)")
    for k, r in res['shapes'].items():
        for a, t in r['train'].items():
            print(f"{k:10s} {a:10s} train {t['ms_median']} ms [{t['ms_min']}-{t['ms_max']}]")
        print(f"{k:10s} GHMC histogram + weights {r['ghmc_bin_weights']['ms_median']} ms over {r['ghmc_logits_mb']} MB of logits, "
              f"GHMR {r['ghmr_bin_weights']['ms_median']} ms")
    print(json.dumps(res))


if __name__ == '__main__':
    main()
