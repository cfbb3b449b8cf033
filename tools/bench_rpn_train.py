"""Times the RPN training path at BASELINE.json configs[3]'s shape: 16 tiles of 640 x 512 (w x h), FPN strides 4-64, 3 anchors per cell
(81 840 anchors per tile), 256 feature channels, GT_PER_TILE small boxes per tile.  Three arms alternate in one process:
  loss       RPNHead.loss + backward from the output maps (targets, sampling, losses and their gradients: the ptb_rpn_* kernels)
  step       the whole RPN training step: forward of the three convs on the five levels, loss, backward
  reference  the reference's op sequence (oracle/rpn_loss.py: AnchorHead.get_targets + loss restated with torch ops) on the same GPU,
             from the same output maps, + backward
Prints the median and min-max of each arm over --iters timed calls, with the card name and power limit read in the same call.
--profile (a separate run, profiler on) splits the loss arm instead: RPNHead.get_targets alone and the loss sums (forward + backward)
alone, host clock around synchronised calls, and from torch.profiler the device time of the kernels per call, by kernel name.
    python tools/bench_rpn_train.py [--iters 20] [--gt 24] [--profile]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import rpn_loss as orl  # noqa: E402


def card():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--gt', type=int, default=24)
    ap.add_argument('--channels', type=int, default=256)
    ap.add_argument('--profile', action='store_true')
    a = ap.parse_args()
    from pointtinybenchmark_b200.rpn import RPNHead
    assert torch.cuda.is_available(), 'needs a CUDA device'
    dev = torch.device('cuda:0')
    B, H, W = 16, 512, 640
    g = torch.Generator().manual_seed(0)
    kw = orl.head_kwargs('tinyperson')
    kw.update(in_channels=a.channels, feat_channels=a.channels)
    head = RPNHead(**kw, train_cfg=orl.TRAIN).to(dev)
    feats = [torch.randn(B, a.channels, H // s, W // s, generator=g).to(dev) for s in orl.STRIDES]
    gts = [orl._boxes(g, a.gt, H, W, 4.0, 32.0).to(dev) for _ in range(B)]
    metas = [dict(img_shape=(H, W, 3), pad_shape=(H, W, 3)) for _ in range(B)]
    with torch.no_grad():
        maps = head(feats)
    maps = [[m.detach().clone() for m in lvl] for lvl in maps]
    ref_kw, ref_train = orl.head_kwargs('tinyperson'), orl.TRAIN

    def arm_loss():
        cls = [m.requires_grad_(True) for m in maps[0]]
        reg = [m.requires_grad_(True) for m in maps[1]]
        losses = head.loss(cls, reg, gts, metas)
        sum(sum(v) for v in losses.values()).backward()

    def arm_step():
        head.zero_grad(set_to_none=True)
        losses = head.forward_train(feats, metas, gts)
        sum(sum(v) for v in losses.values()).backward()

    def arm_reference():
        cls = [m.requires_grad_(True) for m in maps[0]]
        reg = [m.requires_grad_(True) for m in maps[1]]
        losses, _ = orl.loss(cls, reg, gts, metas, None, ref_kw, ref_train)
        sum(sum(v) for v in losses.values()).backward()

    if a.profile:
        return profile(head, maps, gts, metas, a)
    arms = dict(loss=arm_loss, step=arm_step, reference=arm_reference)
    times = {k: [] for k in arms}
    for it in range(a.iters + 2):
        for k, fn in arms.items():
            torch.manual_seed(it)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            if it >= 2:                                  # two warm-up rounds
                times[k].append((time.perf_counter() - t0) * 1e3)
    res = dict(card=card(), tiles=B, tile_wh=[W, H], anchors_per_tile=sum((H // s) * (W // s) * 3 for s in orl.STRIDES),
               gt_per_tile=a.gt, channels=a.channels, iters=a.iters,
               ms={k: dict(median=round(float(np.median(v)), 3), min=round(min(v), 3), max=round(max(v), 3)) for k, v in times.items()})
    print(json.dumps(res))


def profile(head, maps, gts, metas, a):
    from torch.profiler import ProfilerActivity, profile as tprofile
    from pointtinybenchmark_b200.rpn import _RPNLevelSums
    sizes = [tuple(m.shape[-2:]) for m in maps[0]]
    dev = maps[0][0].device

    def targets():
        return head.get_targets(sizes, gts, metas, device=dev)

    def sums(tg):
        s = _RPNLevelSums.apply(tg, *[m.requires_grad_(True) for m in maps[0] + maps[1]])
        s.sum().backward()

    def clock(fn, n):
        out = []
        for i in range(n + 2):
            torch.manual_seed(i)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            if i >= 2:
                out.append((time.perf_counter() - t0) * 1e3)
        return round(float(np.median(out)), 3)

    tg = targets()
    res = dict(card=card(), gt_per_tile=a.gt, iters=a.iters, host_ms_median=dict(get_targets=clock(targets, a.iters),
                                                                              loss_sums_fwd_bwd=clock(lambda: sums(tg), a.iters)))
    n = 5
    for name, fn in (('get_targets', targets), ('loss_sums_fwd_bwd', lambda: sums(tg))):
        torch.cuda.synchronize()
        with tprofile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for i in range(n):
                torch.manual_seed(i)
                fn()
            torch.cuda.synchronize()
        kern = {}
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA:
                k = kern.setdefault(e.name, [0.0, 0])
                k[0] += e.device_time_total / 1e3 / n
                k[1] += 1
        top = sorted(kern.items(), key=lambda kv: -kv[1][0])[:8]
        res[name] = dict(device_ms_per_call=round(sum(v[0] for v in kern.values()), 3),
                         device_ops_per_call=round(sum(v[1] for v in kern.values()) / n, 1),
                         top=[dict(name=k[:90], ms=round(v[0], 3), count=v[1] // n) for k, v in top])
    print(json.dumps(res))


if __name__ == '__main__':
    main()
