"""HungarianAssignerV2 cost matrix + matching per batch at bench.py's p2p_hungarian shape: 16 images x 16 800 proposals x 100 GTs,
80 classes, topk_k 5, the same seeded inputs.  Times, with CUDA events (median of --iters calls after --warmup), for
  shipped   FocalLossCost(weight 2) + DisCostV2(p=1, weight 0.1)                  ptb_p2p_cost_matrix (the shipped configs)
  paper     ClassificationCostV2(use_sigmoid=False, weight 2) + DisCostV2(p=2, weight 5e-2) on 81 columns (a softmax head)
  zero_l1   ZeroCost + DisCostV2(p=1, weight 0.1)
each the per-image cost matrices and one ptb_hungarian_v2_batch.  Prints the card's name and power limit, then one JSON line.
Writes nothing.

    python tools/bench_p2p_match_costs.py [--iters 20] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pointtinybenchmark_b200 import assigners, ops  # noqa: E402

SETS = {
    'shipped': ([dict(type='FocalLossCost', weight=2.0)], [dict(type='DisCostV2', weight=0.1)]),
    'paper': ([dict(type='ClassificationCostV2', use_sigmoid=False, weight=2.0)], [dict(type='DisCostV2', weight=5e-2, p=2)]),
    'zero_l1': ([dict(type='ZeroCost')], [dict(type='DisCostV2', weight=0.1)]),
}


def card():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0) + ', power limit unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_p2p_match_costs: no CUDA device')
    dev = torch.device('cuda:0')
    # bench.py's p2p_hungarian inputs (seed 9): a 100 x 168 map at stride 8, proposals near the cell centres, GTs in 1333 x 800
    B, H, W, n, C, stride = 16, 100, 168, 100, 80, 8
    Q = H * W
    g = torch.Generator().manual_seed(9)
    cls = (torch.randn(B, Q, C, generator=g) * 1.5 - 3.0).to(dev)
    xs, ys = (torch.arange(Q) % W).float() * stride, (torch.arange(Q) // W).float() * stride
    prop = (torch.stack([xs, ys], 1)[None] + torch.randn(B, Q, 2, generator=g) * 4).to(dev).contiguous()
    gts = (torch.rand(B, n, 2, generator=g) * torch.tensor([1333., 800.])).to(dev)
    labels = torch.randint(0, C, (B, n), generator=g).int().to(dev)
    cls81 = torch.cat([cls, torch.full((B, Q, 1), 2.0, device=dev)], -1).contiguous()      # a background column for the softmax head
    cost = torch.empty(B * Q * n, device=dev)
    gi = torch.zeros(B * Q, dtype=torch.int64, device=dev)
    img_shape = (800, 1333, 3)
    print('card:', card(), flush=True)
    res = dict(shape=f'{B} x ({Q} proposals x {n} GTs), {C} classes, topk_k 5', iters=args.iters)
    for name, (cc, rc) in SETS.items():
        terms = assigners.match_cost_terms(cc, rc)
        c = cls81 if name == 'paper' else cls

        def assign():
            for b in range(B):
                assigners.cost_matrix(c[b], prop[b], None, gts[b], labels[b], terms, img_shape, out=cost[b * Q * n:(b + 1) * Q * n])
            gi.zero_()
            return ops.hungarian_v2_batch(cost, [(Q, n)] * B, 5, gi, [b * Q for b in range(B)])
        for _ in range(args.warmup):
            assign()
        torch.cuda.synchronize()
        ts = []
        for _ in range(args.iters):
            a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            st = assign()
            e.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(e))
        ts.sort()
        res[name] = dict(ms_per_batch_median=ts[len(ts) // 2], ms_min=ts[0], status_ok=bool(int(st.max()) == 0),
                         positives=int((gi > 0).sum()), path='ptb_p2p_cost_matrix' if assigners.is_focal_l1_pair(terms)
                         else 'ptb_p2p_cost_matrix_terms')
    print(json.dumps(res))


if __name__ == '__main__':
    main()
