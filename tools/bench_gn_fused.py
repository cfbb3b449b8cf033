"""The tower conv with GroupNorm + ReLU applied inside the conv kernel (ops.conv3x3_c256_f16_gn) against the explicit unfused op
sequence it replaced (ops.conv3x3_c256_f16, then ops.gn_relu_apply_f16 / gn_relu_apply), in one process:
  tower   the four-layer cls tower of CPRHead (want='f16pair', what simple_test runs), batch 8 of 256 x 100 x 168
  step    CPRHead.simple_test at bench.py's headline shape and inputs
The unfused arm runs the same head with ops.conv3x3_c256_f16_gn swapped for the two-kernel sequence.  A round times both arms
(CUDA events around `--calls` calls each, two input sets larger than L2 rotating); rounds alternate which arm goes first.  Prints
one JSON line: the median and min - max per call of each arm, the card, its power limit and the SM clock sampled while timing.

    python tools/bench_gn_fused.py [--rounds N] [--calls N]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import bench  # noqa: E402
from bench_half_inputs import card  # noqa: E402
from pointtinybenchmark_b200 import cpr_head, ops  # noqa: E402,F401
from pointtinybenchmark_b200.layers import tower  # noqa: E402
from pointtinybenchmark_b200.registry import build_head  # noqa: E402

FUSED = ops.conv3x3_c256_f16_gn


def unfused(x_h, x_l, w_h, w_l, out_scale, dev_out_scale, gamma, beta, eps=1e-5, overflow_flag=None, out='f16pair'):
    """the two-kernel sequence with the fused op's signature and results."""
    y, st = ops.conv3x3_c256_f16(x_h, x_l, w_h, w_l, out_scale, dev_out_scale)
    if out == 'fp32':
        return ops.gn_relu_apply(y, st, gamma, beta, 32, eps, True, split=False), None, y, st
    h, l = ops.gn_relu_apply_f16(y, st, gamma, beta, 32, eps, True, overflow_flag)
    return h, l, y, st


def timed(arm, fn, calls):
    ops.conv3x3_c256_f16_gn = FUSED if arm == 'fused' else unfused
    s, e = torch.cuda.Event(True), torch.cuda.Event(True)
    s.record()
    for i in range(calls):
        fn(i)
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=9)
    ap.add_argument('--calls', type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device (there is no CPU fallback)')
    if args.rounds < 7:
        raise SystemExit('--rounds must be at least 7')
    dev = torch.device('cuda:0')
    head = build_head(bench.head_cfg()).to(dev).eval()
    sd = head.state_dict()
    sd.update(bench.head_weights())
    head.load_state_dict(sd)
    sets = []
    for i in range(2):
        x, gtb, gtl, aid, metas = bench.synth_batch(bench.CFG['B'], 1234 + i)
        sets.append((x.to(dev).contiguous(memory_format=torch.channels_last), [t.to(dev) for t in gtb], [t.to(dev) for t in gtl],
                     [t.to(dev) for t in aid], metas))

    def tower_fn(i):
        with torch.no_grad():
            return tower(head.cls_convs, sets[i % 2][0], None, want='f16pair')

    def step_fn(i):
        x, gtb, gtl, aid, metas = sets[i % 2]
        with torch.no_grad():
            return head.simple_test((x,), metas, gt_bboxes=gtb, gt_labels=gtl, gt_anns_id=aid)

    arms = ('fused', 'unfused')
    out = dict(card=card(), rounds=args.rounds, calls_per_round=args.calls, unit='ms per call')
    sampler = bench.ClockSampler(torch.cuda.current_device())
    sampler.start()
    t0 = time.perf_counter()
    for name, fn in (('tower', tower_fn), ('step', step_fn)):
        for a in arms:                                   # warm-up: module loads, allocator, packed-weight caches
            timed(a, fn, 3)
        ts = {a: [] for a in arms}
        for r in range(args.rounds):
            for a in (arms if r % 2 == 0 else arms[::-1]):
                ts[a].append(timed(a, fn, args.calls))
        out[name] = {a: dict(median_ms=float(np.median(v)), min_ms=float(min(v)), max_ms=float(max(v))) for a, v in ts.items()}
        out[name]['saved_ms_median'] = out[name]['unfused']['median_ms'] - out[name]['fused']['median_ms']
    ops.conv3x3_c256_f16_gn = FUSED
    out['clocks'] = sampler.stop(t0, time.perf_counter())
    print(json.dumps(out))


if __name__ == '__main__':
    main()
