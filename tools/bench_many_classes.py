"""CPRHead at many classes: the training step and simple_test at the headline shape (8 images of 256 x 100 x 168, stride 8, 500 GT
points per image: G = 4000 ring bags of radius 8, K = 289) for 80, 365 (Objects365) and 1203 (LVIS) classes.

  train        forward_train (towers + loss) + backward, timed with CUDA events; median and min over --iters steps, peak memory
  simple_test  towers + class-logit map + fused refine under torch.no_grad; median and min, peak memory
  bwd_gemms    the logit map's two backward GEMMs (dW, dX) on their own at the step's shape (M = 134 400 pixels x LD columns x 256), on
               the kernels the head runs them on (the tensor cores: dW as one wgrad up to LD 256, in column slices above; dX one conv),
               with the fp32 FFMA kernels next to them for comparison
The (G, K, LD) bag-logit tensor of the loss (G * K * LD * 4 B, LD from cpr_head.loss_bwd_plan) is reported with each class count.
Prints the card's name and power limit, then one JSON line.  Writes nothing.

    python tools/bench_many_classes.py [--iters 20] [--warmup 3] [--classes 80,365,1203] [--images 8]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import bench  # noqa: E402  (headline shape, synthetic batch and weights)
from pointtinybenchmark_b200 import cpr_head, ops  # noqa: E402,F401  (registers the head)
from pointtinybenchmark_b200.registry import build_head  # noqa: E402


def card():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0) + ', power limit unknown'


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return dict(ms_median=round(ts[len(ts) // 2], 3), ms_min=round(ts[0], 3), peak_gb=round(torch.cuda.max_memory_allocated() / 1e9, 2))


def weights(N, seed=7):
    w = bench.head_weights(seed)
    g = torch.Generator().manual_seed(seed + N)
    C = bench.CFG['C']
    w['cls_out.weight'] = torch.randn(N, C, generator=g) * 0.01 * 8.0
    w['cls_out.bias'] = torch.full((N,), -float(np.log(99.0)))
    w['ins_out.weight'] = torch.randn(N, C, generator=g) * 0.01 * 8.0
    w['ins_out.bias'] = torch.zeros(N)
    return w


def run(N, B, iters, warmup, dev):
    x, gtb, _, aid, metas = bench.synth_batch(B, 11)
    g = torch.Generator().manual_seed(N)
    gtl = [torch.randint(0, N, (len(b),), generator=g).to(dev) for b in gtb]
    x = x.to(dev).contiguous(memory_format=torch.channels_last)
    gtb = [t.to(dev) for t in gtb]
    aid = [t.to(dev) for t in aid]
    cfg = bench.head_cfg()
    cfg['num_classes'] = N
    head = build_head(cfg).to(dev)
    sd = head.state_dict()
    sd.update({k: v.to(dev) for k, v in weights(N).items()})
    head.load_state_dict(sd, strict=True)
    G, K = sum(len(b) for b in gtb), 289
    LD = 2 * cpr_head.loss_bwd_plan(N, K, True, True)[0]
    out = dict(G=G, K=K, LD=LD, bag_logits_gb=round(G * K * LD * 4 / 1e9, 2))
    head.train()

    def step():
        head.zero_grad(set_to_none=True)
        losses = head.forward_train([x], metas, gtb, gtl)
        sum(v for k, v in losses.items() if 'loss' in k).backward()
    out['train'] = timed(step, iters, warmup)
    head.eval()

    def infer():
        with torch.no_grad():
            head.simple_test((x,), metas, gt_bboxes=gtb, gt_labels=gtl, gt_anns_id=aid)
    out['simple_test'] = timed(infer, iters, warmup)
    del head
    M, C = x.shape[0] * x.shape[2] * x.shape[3], x.shape[1]
    xr = torch.randn(M, C, device=dev)
    dy = torch.randn(M, LD, device=dev)
    wcat = torch.randn(LD, C, device=dev)
    xh, xl, xinv = ops.split_f16(xr.view(x.shape[0], x.shape[2], x.shape[3], C), auto_scale=True)
    dyv = dy.view(x.shape[0], x.shape[2], x.shape[3], LD)
    wt = ops.conv_tc_pack_weight_f16(wcat.t().contiguous(), 1)

    def tc_dw():
        dh, dl, dinv = ops.split_f16(dyv, auto_scale=True)
        return ops.conv_tc_wgrad_f16(dh, dl, xh, xl, 1, 1.0, dinv, xinv)

    def tc_dx():
        dh, dl, dinv = ops.split_f16(dyv, auto_scale=True)
        return ops.conv_tc_f16(dh, dl, wt, 1, C, dev_out_scale=dinv, ldy=C)
    out['bwd_gemms'] = dict(path='wgmma', dW_ms=timed(tc_dw, iters, warmup)['ms_median'], dX_ms=timed(tc_dx, iters, warmup)['ms_median'],
                            ffma_dW_ms=timed(lambda: ops.linear_rows_bwd_w(dy, xr), iters, warmup)['ms_median'],
                            ffma_dX_ms=timed(lambda: ops.linear_rows_bwd_x(dy, wcat), iters, warmup)['ms_median'],
                            gflop=round(2 * 2 * M * LD * C / 1e9, 1))
    del xr, dy, wcat, xh, xl, dyv
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--classes', default='80,365,1203')
    ap.add_argument('--images', type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_many_classes: no CUDA device')
    dev = torch.device('cuda:0')
    print('card:', card(), flush=True)
    res = dict(shape=f'B={args.images} 100x168x256 stride 8, 500 points / image, K=289', iters=args.iters)
    for N in (int(n) for n in args.classes.split(',')):
        res[f'N={N}'] = run(N, args.images, args.iters, args.warmup, dev)
        print(f'N={N}: {json.dumps(res[f"N={N}"])}', flush=True)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
