"""Times StandardRoIHead (bbox branch) on the GPU; prints the card's name and power limit with the timings.

    python tools/bench_roi_head.py [--iters 20] [--profile]

Arms, alternating in one process, median and min-max of --iters:
  train      forward_train + backward at 16 TinyPerson tiles of 640 x 512, 1 000 proposals and 24 GTs per tile, 512 sampled RoIs per tile
  test       simple_test at that shape (1 class)
  test80     simple_test on 8 images of 1333 x 800, 1 000 proposals each, 80 classes, max_per_img 100, seeded fc_cls / fc_reg scaled so
             that about a thousand (RoI, class) candidates per image pass score_thr (the tool prints how many detections result)
  ref_train  the reference's op sequence after sampling, on the same GPU and the same sampled RoIs: per level nonzero + RoIAlign, the
             same nn.Linear layers, F.cross_entropy and the L1 loss, backward.  mmcv's CUDA RoIAlign is not available here, so
             torchvision.ops.roi_align(aligned=True) stands in for it.
--profile runs each of the three head arms once under torch.profiler and splits the CUDA time into RoIAlign forward / backward,
targets (assignment, ranks, targets), losses, decode + NMS and the FC GEMMs."""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as e:          # the timings still stand; say why the card line is missing
        return f'(nvidia-smi unavailable: {e})'


def inputs(seed, B, H, W, n_gt, n_prop, dev):
    g = torch.Generator().manual_seed(seed)
    feats = [torch.randn(B, 256, H // s, W // s, generator=g).to(dev) for s in (4, 8, 16, 32, 64)]
    gts, labels, props = [], [], []
    for _ in range(B):
        c = torch.rand(n_gt, 2, generator=g) * torch.tensor([W, H])
        s = torch.rand(n_gt, 2, generator=g) * 40 + 6
        gt = torch.cat([c - s / 2, c + s / 2], 1).clamp(min=0)
        c = torch.rand(n_prop, 2, generator=g) * torch.tensor([W, H])
        s = torch.rand(n_prop, 2, generator=g) * 150 + 4
        p = torch.cat([c - s / 2, c + s / 2], 1).clamp(min=0)
        m = n_prop // 3
        p[:m] = gt[torch.randint(0, n_gt, (m,), generator=g)] + torch.randn(m, 4, generator=g) * 2
        gts.append(gt.to(dev)); labels.append(torch.zeros(n_gt, dtype=torch.long, device=dev))
        props.append(torch.cat([p, torch.rand(n_prop, 1, generator=g)], 1).to(dev))
    metas = [dict(img_shape=(H, W, 3), pad_shape=(H, W, 3), scale_factor=np.ones(4, np.float32)) for _ in range(B)]
    return feats, gts, labels, props, metas


def make_head(num_classes, dev):
    from pointtinybenchmark_b200.roi_head import StandardRoIHead
    return StandardRoIHead(
        bbox_roi_extractor=dict(type='SingleRoIExtractor', roi_layer=dict(type='RoIAlign', output_size=7, sampling_ratio=0), out_channels=256,
                                featmap_strides=[4, 8, 16, 32]),
        bbox_head=dict(type='Shared2FCBBoxHead', in_channels=256, fc_out_channels=1024, roi_feat_size=7, num_classes=num_classes,
                       bbox_coder=dict(type='DeltaXYWHBBoxCoder', target_means=[0.] * 4, target_stds=[0.1, 0.1, 0.2, 0.2]),
                       loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0), loss_bbox=dict(type='L1Loss', loss_weight=1.0)),
        train_cfg=dict(assigner=dict(type='MaxIoUAssigner', pos_iou_thr=0.5, neg_iou_thr=0.5, min_pos_iou=0.5, match_low_quality=False,
                                     ignore_iof_thr=-1),
                       sampler=dict(type='RandomSampler', num=512, pos_fraction=0.25, neg_pos_ub=-1, add_gt_as_proposals=True), pos_weight=-1),
        test_cfg=dict(score_thr=0.05, nms=dict(type='nms', iou_threshold=0.5), max_per_img=-1 if num_classes == 1 else 100)).to(dev)


def ref_train(head, feats, rois, labels, bt, bw):
    """the reference's sequence after sampling (single_level_roi_extractor.py, convfc_bbox_head.py, bbox_head.py:261-306)"""
    import torchvision
    ex = head.bbox_roi_extractor
    scale = torch.sqrt((rois[:, 3] - rois[:, 1]) * (rois[:, 4] - rois[:, 2]))
    lv = torch.floor(torch.log2(scale / 56 + 1e-6)).clamp(0, 3).long()
    y = feats[0].new_zeros(rois.shape[0], 256, 7, 7)
    for i, s in enumerate(ex.featmap_strides):
        inds = (lv == i).nonzero(as_tuple=False).squeeze(1)
        if inds.numel():
            y[inds] = torchvision.ops.roi_align(feats[i], rois[inds], 7, 1.0 / s, 0, aligned=True)
        else:
            y = y + feats[i].sum() * 0.
    cls, reg = head.bbox_head(y)
    loss_cls = F.cross_entropy(cls, labels, reduction='sum') / max(float(rois.shape[0]), 1.)
    pos = labels < head.bbox_head.num_classes
    p = reg.view(reg.shape[0], -1, 4)[pos, labels[pos]]
    loss_bbox = (torch.abs(p - bt[pos]) * bw[pos]).sum() / bt.shape[0]
    (loss_cls + loss_bbox).backward()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--profile', action='store_true')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_roi_head needs a CUDA device')
    dev = torch.device('cuda:0')
    print('card:', card(), flush=True)
    feats, gts, labels, props, metas = inputs(1, 16, 512, 640, 24, 1000, dev)
    f80, _, _, p80, m80 = inputs(2, 8, 800, 1344, 10, 1000, dev)
    head, head80 = make_head(1, dev), make_head(80, dev)
    # fc_cls / fc_reg at the spread of a trained head: at the reference init every one of 81 softmax scores sits near 1 / 81, below
    # score_thr, and the arm would time an NMS without candidates
    torch.manual_seed(17)
    head80.bbox_head.init_weights()
    with torch.no_grad():
        head80.bbox_head.fc_cls.weight.normal_(0.0, 0.1)
        head80.bbox_head.fc_reg.weight.normal_(0.0, 0.05)
        n80 = sum(sum(len(c) for c in r) for r in head80.simple_test(f80, p80, m80))
    print(f'test80: {n80} detections over the 8 images (max_per_img 100)', flush=True)
    x = [f.requires_grad_(True) for f in feats]
    torch.manual_seed(0)
    rois, lab, _, bt, bw, _ = head.get_targets(props, gts, labels)

    def train():
        head.zero_grad(set_to_none=True)
        for f in x:
            f.grad = None
        l = head.forward_train(x, metas, props, gts, labels)
        (l['loss_cls'] + l['loss_bbox']).backward()

    def test():
        with torch.no_grad():
            head.simple_test(feats, props, metas)

    def test80():
        with torch.no_grad():
            head80.simple_test(f80, p80, m80)

    def ref():
        head.zero_grad(set_to_none=True)
        for f in x:
            f.grad = None
        ref_train(head, x, rois, lab, bt, bw)

    arms = dict(train=train, test=test, test80=test80, ref_train=ref)
    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        for fn in arms.values():
            fn()
        torch.cuda.synchronize()
        cats = [('roi_align_fwd', ('roi_align_fwd_kernel',)), ('roi_align_bwd', ('roi_align_bwd_kernel',)),
                ('targets', ('roi_targets_kernel', 'rpn_candidate_kernel', 'max_iou', 'assign')),
                ('losses', ('loss_sum_kernel', 'softmax_ce', 'roi_accuracy')), ('decode+nms', ('roi_decode', 'nms')),
                ('fc_gemm', ('gemm', 'sgemm', 'cutlass', 'xmma', 'ampere', 'sm90'))]
        for name in ('train', 'test', 'test80'):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                arms[name]()
                torch.cuda.synchronize()
            tot, split = 0.0, {c: 0.0 for c, _ in cats}
            split['other'] = 0.0
            for e in prof.key_averages():
                t = e.device_time_total if hasattr(e, 'device_time_total') else e.cuda_time_total
                if t <= 0:
                    continue
                tot += t
                key = next((c for c, pats in cats if any(p in e.key for p in pats)), 'other')
                split[key] += t
            print(f'profile {name}: CUDA time {tot / 1e3:.2f} ms: ' + ', '.join(f'{k} {v / 1e3:.2f} ms ({100 * v / max(tot, 1e-9):.0f} %)'
                                                                       for k, v in split.items()), flush=True)
        return
    for fn in arms.values():                       # warm-up of every shape
        fn(); fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(a.iters):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[k].append((time.perf_counter() - t0) * 1e3)
    for k, v in times.items():
        print(f'{k}: median {np.median(v):.2f} ms (min {min(v):.2f}, max {max(v):.2f}) over {len(v)}', flush=True)
    print('ref_train: torchvision.ops.roi_align(aligned=True) stands in for mmcv RoIAlign; it starts from the sampled RoIs '
          '(no assignment or sampling)', flush=True)


if __name__ == '__main__':
    main()
