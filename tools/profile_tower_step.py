"""Kernel times of one CPRHead.simple_test step at bench.py's headline shape (8 x 256 x 100 x 168), from torch.profiler with
CUDA activities: every launch of the step in order, with its name and device time, and the totals per kernel name.  Prints one
JSON line with the card, its power limit and SM clock; writes the Chrome trace to OUT_DIR/tower_step.pt.trace.json.

    python tools/profile_tower_step.py [OUT_DIR]        (default: <temp dir>/ptb_profile)
"""
import json
import os
import sys
import tempfile
import time

import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import bench  # noqa: E402
from bench_half_inputs import card  # noqa: E402
from pointtinybenchmark_b200 import cpr_head  # noqa: E402,F401
from pointtinybenchmark_b200.registry import build_head  # noqa: E402


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else os.path.join(tempfile.gettempdir(), 'ptb_profile')
    os.makedirs(out_dir, exist_ok=True)
    dev = torch.device('cuda:0')
    head = build_head(bench.head_cfg()).to(dev).eval()
    sd = head.state_dict()
    sd.update(bench.head_weights())
    head.load_state_dict(sd)
    x, gtb, gtl, aid, metas = bench.synth_batch(bench.CFG['B'], 1234)
    x = x.to(dev).contiguous(memory_format=torch.channels_last)
    gtb, gtl, aid = [t.to(dev) for t in gtb], [t.to(dev) for t in gtl], [t.to(dev) for t in aid]

    def step():
        with torch.no_grad():
            return head.simple_test((x,), metas, gt_bboxes=gtb, gt_labels=gtl, gt_anns_id=aid)

    for _ in range(5):
        step()
    torch.cuda.synchronize()
    sampler = bench.ClockSampler(torch.cuda.current_device())
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    prof.export_chrome_trace(os.path.join(out_dir, 'tower_step.pt.trace.json'))
    events = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA), key=lambda e: e.time_range.start)
    launches = [dict(name=e.name[:120], us=round(e.device_time, 2)) for e in events]
    totals = {}
    for e in launches:
        totals[e['name']] = round(totals.get(e['name'], 0.0) + e['us'], 2)
    sampler.start()                      # the SM clock while the same step runs unprofiled
    t0 = time.perf_counter()
    for _ in range(20):
        step()
    torch.cuda.synchronize()
    clocks = sampler.stop(t0, time.perf_counter())
    gn = [e['us'] for e in launches if 'gn_relu_apply_f16' in e['name']]
    conv = [e['us'] for e in launches if 'conv_tc_kernel' in e['name']]
    print(json.dumps(dict(card=card(), clocks=clocks, gn_relu_apply_f16_us=gn, gn_relu_apply_f16_total_us=round(sum(gn), 2),
                          conv_tc_us=conv, step_kernels_total_us=round(sum(e['us'] for e in launches), 2), n_launches=len(launches),
                          totals_us=dict(sorted(totals.items(), key=lambda kv: -kv[1])), launches=launches)))


if __name__ == '__main__':
    main()
