"""P2PHead at many classes, at the reference class's own defaults (4 point anchors per cell, CrossEntropyLoss(use_sigmoid=True) +
MSELoss): 16 images of 256 x 100 x 168 at stride 8 (67 200 proposals per image), for 80, 365 (Objects365) and 1203 (LVIS) classes,
i.e. a cls_out of 320, 1460 and 4812 channels.

  simple_test  towers + output convs + decode / top-k / NMS under torch.no_grad
  train        forward_train (towers + output convs + matching + loss) + backward, 20 GT points per image
  cls_out      the output conv alone, forward + backward (dX, dW, db) at 1460 and 4812 channels: the tensor-core path the head runs
               above 512 channels (layers.wide_out_conv) against torch.nn.functional.conv2d on cuDNN fp32 with TF32 off (a local
               cudnn.flags context, as the head uses for its narrow output convs), the two arms alternating call by call
Each: CUDA events around each call (which ends in a device synchronise), --iters timed calls after --warmup, median and min-max in ms,
and the peak memory of the timed calls.  Prints the card's name, power limit and SM clock, then one JSON line.  Writes nothing.

    python tools/bench_p2p_many_classes.py [--iters 20] [--warmup 3] [--classes 80,365,1203] [--widths 1460,4812]
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pointtinybenchmark_b200 import p2p_head  # noqa: E402,F401  (registers the head)
from pointtinybenchmark_b200.layers import wide_out_conv  # noqa: E402
from pointtinybenchmark_b200.registry import build_head  # noqa: E402

B, C, H, W, STRIDE, N_GT = 16, 256, 100, 168, 8, 20
PAD_HW, IMG_HW = (800, 1344), (800, 1333)
TRAIN_CFG = dict(neg_weight=1.0, assigner=dict(type='HungarianAssignerV2', cls_costs=dict(type='FocalLossCost', weight=2.0),
                                               reg_costs=dict(type='DisCostV2', weight=0.1, norm_with_img_wh=False), topk_k=5),
                 sampler=dict(type='PseudoSampler'))
TEST_CFG = dict(nms_pre=1000, min_bbox_size=0, score_thr=0.05, pseudo_wh=(32, 32), nms=dict(type='nms', iou_threshold=0.5),
                max_per_img=100)


def card():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0) + ', power limit and clocks unknown'


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def summary(ts, peak=None):
    ts = sorted(ts)
    out = dict(ms_median=round(ts[len(ts) // 2], 3), ms_min=round(ts[0], 3), ms_max=round(ts[-1], 3), n=len(ts))
    if peak is not None:
        out['peak_gb'] = round(peak / 1e9, 2)
    return out


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    ts = [event_ms(fn) for _ in range(iters)]
    return summary(ts, torch.cuda.max_memory_allocated())


def head_step(N, x, metas, gtb, iters, warmup, dev):
    g = torch.Generator().manual_seed(N)
    gtl = [torch.randint(0, N, (N_GT,), generator=g).to(dev) for _ in range(B)]
    cfg = dict(type='P2PHead', norm_cfg=dict(type='GN', num_groups=32, requires_grad=True), num_classes=N, in_channels=C,
               feat_channels=C, stacked_convs=4, strides=[STRIDE], train_cfg=TRAIN_CFG, test_cfg=TEST_CFG)
    head = build_head(cfg).to(dev)
    out = dict(cls_out_channels=head.cls_out.out_channels)
    head.eval()

    def infer():
        with torch.no_grad():
            head.simple_test((x,), metas)
    out['simple_test'] = timed(infer, iters, warmup)
    head.train()

    def step():
        head.zero_grad(set_to_none=True)
        ls = head.forward_train((x,), metas, gtb, gtl)
        (sum(ls['loss_cls']) + sum(ls['loss_pts'])).backward()
    out['train'] = timed(step, iters, warmup)
    del head
    torch.cuda.empty_cache()
    return out


def cls_out_arms(n_out, iters, warmup, dev):
    """forward + backward of the output conv alone: the tensor-core path and cuDNN fp32, alternating call by call."""
    g = torch.Generator().manual_seed(n_out)
    x = torch.relu(torch.randn(B, C, H, W, generator=g)).to(dev).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    conv = nn.Conv2d(C, n_out, 3, padding=1).to(dev)
    with torch.no_grad():
        conv.weight.normal_(0.0, 0.01)
    gy = torch.randn(B, n_out, H, W, device=dev).contiguous(memory_format=torch.channels_last)

    def tc():
        x.grad = conv.weight.grad = conv.bias.grad = None
        wide_out_conv(conv, x).backward(gy)

    def cudnn():
        x.grad = conv.weight.grad = conv.bias.grad = None
        with torch.backends.cudnn.flags(enabled=True, benchmark=torch.backends.cudnn.benchmark,
                                        deterministic=torch.backends.cudnn.deterministic, allow_tf32=False):
            F.conv2d(x, conv.weight, conv.bias, 1, 1).backward(gy)
    for _ in range(warmup):
        tc(); cudnn()
    torch.cuda.synchronize()
    t_tc, t_dnn = [], []
    for _ in range(iters):
        t_tc.append(event_ms(tc))
        t_dnn.append(event_ms(cudnn))
    tflop = 3 * 2 * 9 * C * n_out * B * H * W / 1e12          # forward, dX and dW: three GEMMs of the same size
    res = dict(tflop=round(tflop, 2), tensor_core=summary(t_tc), cudnn_fp32=summary(t_dnn))
    res['speedup_median'] = round(res['cudnn_fp32']['ms_median'] / res['tensor_core']['ms_median'], 2)
    del x, conv, gy
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--classes', default='80,365,1203')
    ap.add_argument('--widths', default='1460,4812')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_p2p_many_classes: no CUDA device')
    dev = torch.device('cuda:0')
    print('card:', card(), flush=True)
    x = torch.randn(B, C, H, W, generator=torch.Generator().manual_seed(11)).to(dev).contiguous(memory_format=torch.channels_last)
    metas = [dict(pad_shape=PAD_HW + (3,), img_shape=IMG_HW + (3,), scale_factor=[1.0, 1.0, 1.0, 1.0])] * B
    g = torch.Generator().manual_seed(13)
    gtb = []
    for _ in range(B):
        cxy = torch.rand(N_GT, 2, generator=g) * torch.tensor([1300., 780.]) + 10
        gtb.append(torch.cat([cxy - 8, cxy + 8], 1).to(dev))
    res = dict(workload=f'P2PHead reference defaults (4 anchors / cell, CE + MSE), {B} x ({C}x{H}x{W}) stride {STRIDE}, '
                        f'{H * W * 4} proposals per image, {N_GT} GT points per image, random-init weights', iters=args.iters)
    for N in (int(n) for n in args.classes.split(',')):
        res[f'N={N}'] = head_step(N, x, metas, gtb, args.iters, args.warmup, dev)
        print(f'N={N}: {json.dumps(res[f"N={N}"])}', flush=True)
    for n in (int(v) for v in args.widths.split(',')):
        res[f'cls_out_{n}'] = cls_out_arms(n, args.iters, args.warmup, dev)
        print(f'cls_out {n}: {json.dumps(res[f"cls_out_{n}"])}', flush=True)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
