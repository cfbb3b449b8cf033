"""CPRHead training step per positive-bag loss at the headline shape: 8 images of 256 x 100 x 168 (stride 8), 500 GT points per image
(G = 4000 bags), ring bags of radius 8 (K = 289), 80 classes.  The step is forward_train (towers + loss) + backward, timed with CUDA
events, for
  mil_gfocal     MILLoss(loss_type='gfocal_loss')            (the shipped configs; what bench.py's train step runs)
  mil_bce        MILLoss(loss_type='binary_cross_entropy')
  allpos_gfocal  AllPosLoss(loss_type='gfocal_loss')
  allpos_bce     AllPosLoss(loss_type='binary_cross_entropy')
in the default (scatter) backward and, with --deterministic, under torch.use_deterministic_algorithms(True) (tile backward).
Prints the card's name and power limit, then one JSON line.  Writes nothing.

    python tools/bench_cpr_loss_types.py [--iters 20] [--warmup 3] [--deterministic]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import bench  # noqa: E402  (headline shape, synthetic batch and weights)
from pointtinybenchmark_b200 import cpr_head  # noqa: E402,F401  (registers the head)
from pointtinybenchmark_b200.registry import build_head  # noqa: E402

LOSSES = {
    'mil_gfocal': dict(type='MILLoss', binary_ins=False, loss_weight=0.25, loss_type='gfocal_loss'),
    'mil_bce': dict(type='MILLoss', binary_ins=False, loss_weight=0.25, loss_type='binary_cross_entropy'),
    'allpos_gfocal': dict(type='AllPosLoss', binary_ins=False, loss_weight=0.25, loss_type='gfocal_loss'),
    'allpos_bce': dict(type='AllPosLoss', binary_ins=False, loss_weight=0.25, loss_type='binary_cross_entropy'),
}


def card():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0) + ', power limit unknown'


def time_step(name, iters, warmup, dev, x, gtb, gtl, metas, weights):
    cfg = bench.head_cfg()
    cfg['loss_mil'] = LOSSES[name]
    head = build_head(cfg).to(dev)
    sd = head.state_dict()
    sd.update({k: v.to(dev) for k, v in weights.items()})
    head.load_state_dict(sd, strict=True)
    head.train()

    def step():
        head.zero_grad(set_to_none=True)
        losses = head.forward_train([x], metas, gtb, gtl)
        sum(v for k, v in losses.items() if 'loss' in k).backward()
        return losses
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        losses = step()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return dict(ms_median=ts[len(ts) // 2], ms_min=ts[0], pos_loss=float(losses['pos_loss'].detach()), bag_acc=float(losses['bag_acc'][0]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--deterministic', action='store_true')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_cpr_loss_types: no CUDA device')
    dev = torch.device('cuda:0')
    torch.use_deterministic_algorithms(args.deterministic)
    B = 8
    x, gtb, gtl, _, metas = bench.synth_batch(B, 11)
    x = x.to(dev).contiguous(memory_format=torch.channels_last)
    gtb = [t.to(dev) for t in gtb]
    gtl = [t.to(dev) for t in gtl]
    weights = bench.head_weights()
    print('card:', card(), flush=True)
    res = dict(shape=f'B={B} 100x168x256 stride 8, G={sum(len(l) for l in gtl)}, K=289, N=80', deterministic=args.deterministic)
    for name in LOSSES:
        res[name] = time_step(name, args.iters, args.warmup, dev, x, gtb, gtl, metas, weights)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
