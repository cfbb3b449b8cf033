"""What the head costs per step for each dtype a backbone can hand it, four arms interleaved in one process:
  fp32        fp32 feature map (the path bench.py times)
  half+float  what users had to do before the half paths: a half tensor and `.float()` in front of the head (bf16 storage)
  fp16        fp16 feature map straight into the towers (hi operand = the tensor, lo == 0 first conv)
  bf16        bf16 feature map (operand pair split from 2-byte storage)
for three workloads:
  cpr_infer   CPRHead.simple_test, batch 8 of 256 x 100 x 168, 500 points per image (bench.py's headline step and inputs)
  cpr_train   CPRHead.forward_train + backward at the same shape, with the input gradient
  p2p_infer   P2PHead.simple_test at the reference defaults (tools/bench_p2p_defaults.py: 16 x 256 x 100 x 168, 4 anchors per cell)
Each workload rotates two input sets larger than L2.  A round times every arm once (CUDA events around `--calls` calls); rounds
alternate the arms, and the result is the median and min - max over the rounds, per call.  Prints one JSON line with the card, its
power limit and the SM clock sampled while timing.  Reads nothing outside the repository and writes nothing.

    python tools/bench_half_inputs.py [--rounds N] [--calls N] [--skip-train] [--skip-p2p]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import bench  # noqa: E402  (the headline workload: head_cfg, synth_batch, head_weights, ClockSampler)
import bench_p2p_defaults as p2pd  # noqa: E402
from pointtinybenchmark_b200 import cpr_head, p2p_head  # noqa: E402,F401  (register the heads)
from pointtinybenchmark_b200.registry import build_head  # noqa: E402

ARMS = ('fp32', 'half+float', 'fp16', 'bf16')


def arm_inputs(x32):
    """the device tensor each arm starts from (channels-last, as a cuDNN backbone under autocast leaves it) and what it does first."""
    cl = lambda t: t.contiguous(memory_format=torch.channels_last)
    xb = cl(x32.to(torch.bfloat16))
    return {'fp32': (cl(x32), lambda t: t), 'half+float': (xb, lambda t: t.float()), 'fp16': (cl(x32.half()), lambda t: t),
            'bf16': (xb, lambda t: t)}


def interleaved(steps, rounds, calls):
    """steps: {arm: fn(i)}.  -> {arm: dict(median_ms, min_ms, max_ms)} per call."""
    for fn in steps.values():                       # warm every arm: module loads, allocator, packed-weight caches
        for i in range(3):
            fn(i)
    torch.cuda.synchronize()
    ts = {a: [] for a in steps}
    order = list(steps)
    for r in range(rounds):
        for a in order[r % len(order):] + order[:r % len(order)]:
            s, e = torch.cuda.Event(True), torch.cuda.Event(True)
            s.record()
            for i in range(calls):
                steps[a](i)
            e.record()
            torch.cuda.synchronize()
            ts[a].append(s.elapsed_time(e) / calls)
    return {a: dict(median_ms=float(np.median(v)), min_ms=float(min(v)), max_ms=float(max(v))) for a, v in ts.items()}


def card():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i',
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=20)
        name, plimit, cmax = [t.strip() for t in r.stdout.strip().splitlines()[0].split(',')]
        return dict(name=name, power_limit=plimit, sm_clock_max=cmax)
    except Exception as ex:      # the numbers stand without it, but say so
        return dict(name=torch.cuda.get_device_name(), power_limit=f'unknown ({type(ex).__name__})', sm_clock_max='unknown')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=7)
    ap.add_argument('--calls', type=int, default=10)
    ap.add_argument('--skip-train', action='store_true')
    ap.add_argument('--skip-p2p', action='store_true')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device (there is no CPU fallback)')
    if args.rounds < 5:
        raise SystemExit('--rounds must be at least 5')
    dev = torch.device('cuda:0')
    out = dict(card=card(), rounds=args.rounds, calls_per_round=args.calls, unit='ms per call')
    sampler = bench.ClockSampler(torch.cuda.current_device())
    sampler.start()
    t_begin = time.perf_counter()

    # ---- CPRHead at the headline shape
    B = bench.CFG['B']
    head = build_head(bench.head_cfg()).to(dev)
    sd = head.state_dict()
    sd.update(bench.head_weights())
    head.load_state_dict(sd, strict=True)
    sets = []
    for i in range(2):
        x, gtb, gtl, aid, metas = bench.synth_batch(B, 1234 + i)
        sets.append((arm_inputs(x.to(dev)), [t.to(dev) for t in gtb], [t.to(dev) for t in gtl], [t.to(dev) for t in aid], metas))

    def infer(arm):
        def fn(i):
            xs, gtb, gtl, aid, metas = sets[i % 2]
            x, pre = xs[arm]
            with torch.no_grad():
                return head.simple_test((pre(x),), metas, gt_bboxes=gtb, gt_labels=gtl, gt_anns_id=aid)
        return fn

    head.eval()
    out['cpr_infer'] = interleaved({a: infer(a) for a in ARMS}, args.rounds, args.calls)
    out['cpr_infer_input_path'] = {}
    for a in ARMS:
        infer(a)(0)
        out['cpr_infer_input_path'][a] = head.last_input_path

    if not args.skip_train:
        head.train()
        leaves = [{a: xs[a][0].clone().requires_grad_(True) for a in ARMS} for xs, *_ in sets]

        def train(arm):
            def fn(i):
                _, gtb, gtl, _, metas = sets[i % 2]
                x = leaves[i % 2][arm]
                x.grad = None
                head.zero_grad(set_to_none=True)
                losses = head.forward_train((sets[i % 2][0][arm][1](x),), metas, gtb, gtl)
                sum(v for k, v in losses.items() if 'loss' in k).backward()
            return fn
        out['cpr_train'] = interleaved({a: train(a) for a in ARMS}, args.rounds, max(2, args.calls // 3))
        del leaves
    del head, sets
    torch.cuda.empty_cache()

    # ---- P2PHead at the reference defaults
    if not args.skip_p2p:
        cfg = dict(type='P2PHead', norm_cfg=dict(type='GN', num_groups=32, requires_grad=True), num_classes=p2pd.NCLS, in_channels=p2pd.C,
                   feat_channels=p2pd.C, stacked_convs=4, strides=[p2pd.STRIDE], test_cfg=p2pd.TEST_CFG)
        phead = build_head(cfg).to(dev).eval()
        metas = [dict(pad_shape=p2pd.PAD_HW + (3,), img_shape=p2pd.IMG_HW + (3,), scale_factor=[1.0, 1.0, 1.0, 1.0])] * p2pd.B
        psets = [arm_inputs(torch.randn(p2pd.B, p2pd.C, p2pd.H, p2pd.W, generator=torch.Generator().manual_seed(11 + i)).to(dev))
                 for i in range(2)]

        def pinfer(arm):
            def fn(i):
                x, pre = psets[i % 2][arm]
                with torch.no_grad():
                    return phead.simple_test((pre(x),), metas)
            return fn
        out['p2p_infer'] = interleaved({a: pinfer(a) for a in ARMS}, args.rounds, max(2, args.calls // 2))

    out['clocks'] = sampler.stop(t_begin, time.perf_counter())
    print(json.dumps(out))


if __name__ == '__main__':
    main()
