"""Tile testing of one 1920 x 1080 image in 12 tiles of 640 x 512 (TinyPerson Faster R-CNN, 256 channels, fc_out_channels=1024,
1 class): three arms timed alternately in one process, median (min - max) of --runs calls, with the card's name and power limit.
  tile_aug_test   pointtinybenchmark_b200.tile_test.tile_aug_test
  reference ops   the reference's per-tile op sequence on the same GPU (two_stage.py:195-258): per tile merge_aug_proposals with
                  torchvision nms, multi-level RoIAlign with torchvision roi_align, the same Linear layers, delta2bbox, the aug mean,
                  batched_nms, the numpy round trip of bbox2result, then the cross-tile batched_nms (torchvision).  Both arms take
                  the RPN's per-aug proposals from the same RPNHead.
  cross-tile NMS  ptb_batched_nms against torchvision batched_nms alone at 12 000 and 65 536 rows.
--logits realistic gives a few detections per tile (44 for the image, a sparse TinyPerson image); --logits scaled multiplies fc_cls so
that hundreds to a thousand detections per tile pass score_thr.  --profile writes a torch.profiler table.
    python tools/bench_tile_test.py [--runs 20] [--logits realistic|scaled] [--profile OUT_DIR]"""
import argparse
import copy
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torchvision

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pointtinybenchmark_b200 import ops  # noqa: E402
from pointtinybenchmark_b200.roi_head import StandardRoIHead  # noqa: E402
from pointtinybenchmark_b200.rpn import RPNHead  # noqa: E402
from pointtinybenchmark_b200.tile_test import tile_aug_test  # noqa: E402

STRIDES = [4, 8, 16, 32, 64]
TH, TW = 512, 640
OFFSETS = [(x, y) for y in (0, 284, 568) for x in (0, 540, 1080, 1280)]      # 640 x 512 tiles, overlap >= 100, over 1920 x 1080


def build(scaled):
    rpn_cfg = dict(nms_pre=1000, max_per_img=1000, nms=dict(type='nms', iou_threshold=0.7), min_bbox_size=0)
    test = dict(score_thr=0.05, nms=dict(type='nms', iou_threshold=0.5), max_per_img=-1)
    rpn = RPNHead(256, 256, anchor_generator=dict(type='AnchorGenerator', scales=[2], ratios=[0.5, 1.0, 2.0], strides=STRIDES),
                  test_cfg=rpn_cfg).cuda().eval()
    roi = StandardRoIHead(bbox_roi_extractor=dict(type='SingleRoIExtractor', roi_layer=dict(type='RoIAlign', output_size=7, sampling_ratio=0),
                                                  out_channels=256, featmap_strides=STRIDES[:4]),
                          bbox_head=dict(type='Shared2FCBBoxHead', in_channels=256, fc_out_channels=1024, roi_feat_size=7, num_classes=1,
                                         bbox_coder=dict(type='DeltaXYWHBBoxCoder', target_means=[0.] * 4, target_stds=[0.1, 0.1, 0.2, 0.2])),
                          test_cfg=test).cuda().eval()
    g = torch.Generator().manual_seed(0)
    with torch.no_grad():
        for m in (rpn.rpn_conv, rpn.rpn_cls, rpn.rpn_reg):
            m.weight.copy_(torch.randn(m.weight.shape, generator=g) * 0.02)
        rpn.rpn_cls.bias.fill_(-2.0)
        fcc = roi.bbox_head.fc_cls
        fcc.weight.copy_(torch.randn(fcc.weight.shape, generator=g) * (0.3 if scaled else 0.02))
        fcc.bias.copy_(torch.tensor([2.0, 0.0]) if scaled else torch.tensor([-1.0, 2.4]))       # realistic: a few per tile, 44 for the image
    feats = [[torch.randn(1, 256, -(-TH // s), -(-TW // s), generator=g).cuda() for s in STRIDES] for _ in OFFSETS]
    metas = [[dict(img_shape=(TH, TW, 3), pad_shape=(TH, TW, 3), ori_shape=(1080, 1920, 3), scale_factor=np.ones(4, np.float32), flip=False,
                   flip_direction=None, tile_offset=o)] for o in OFFSETS]
    return rpn, roi, feats, metas, rpn_cfg, test


def delta2bbox(rois, d, means, stds, h, w, max_ratio=abs(np.log(16 / 1000))):
    d = d.view(d.shape[0], -1, 4) * d.new_tensor(stds) + d.new_tensor(means)
    px, py = (rois[:, 0] + rois[:, 2]) * 0.5, (rois[:, 1] + rois[:, 3]) * 0.5
    pw, ph = rois[:, 2] - rois[:, 0], rois[:, 3] - rois[:, 1]
    dw, dh = d[..., 2].clamp(-max_ratio, max_ratio), d[..., 3].clamp(-max_ratio, max_ratio)
    gw, gh = pw[:, None] * dw.exp(), ph[:, None] * dh.exp()
    gx, gy = px[:, None] + pw[:, None] * d[..., 0], py[:, None] + ph[:, None] * d[..., 1]
    b = torch.stack([gx - gw * 0.5, gy - gh * 0.5, gx + gw * 0.5, gy + gh * 0.5], -1)
    b[..., 0::2] = b[..., 0::2].clamp(0, w)
    b[..., 1::2] = b[..., 1::2].clamp(0, h)
    return b.view(b.shape[0], -1)


def reference_ops(rpn, roi, feats, metas, rpn_cfg, test):
    """the reference's per-tile sequence with torchvision ops (one aug per tile here: no flip, scale 1)"""
    bh = roi.bbox_head
    all_b, all_l = [], []
    for f, m in zip(feats, metas):
        p = rpn.simple_test_rpn(f, m)[0]
        keep = torchvision.ops.nms(p[:, :4], p[:, 4], rpn_cfg['nms']['iou_threshold'])
        p = p[keep]
        p = p[p[:, 4].sort(descending=True)[1][:rpn_cfg['max_per_img']]]
        rois = torch.cat([p.new_zeros(len(p), 1), p[:, :4]], 1)
        scale = torch.sqrt((rois[:, 3] - rois[:, 1]) * (rois[:, 4] - rois[:, 2]))
        lvl = torch.floor(torch.log2(scale / 56 + 1e-6)).clamp(min=0, max=3).long()
        x = rois.new_zeros(len(rois), 256, 7, 7)
        for i in range(4):
            ix = (lvl == i).nonzero().squeeze(1)
            if len(ix):
                x[ix] = torchvision.ops.roi_align(f[i], rois[ix], 7, 1.0 / STRIDES[i], 0, aligned=True)
        x = x.flatten(1)
        for fc in bh.shared_fcs:
            x = torch.relu(fc(x))
        s = torch.softmax(bh.fc_cls(x), -1)
        b = delta2bbox(rois[:, 1:], bh.fc_reg(x), bh.means, bh.stds, TH, TW)
        b, s = torch.stack([b]).mean(0), torch.stack([s]).mean(0)
        valid = s[:, 0] > test['score_thr']
        bb, ss = b[valid], s[valid, 0]
        k = torchvision.ops.batched_nms(bb, ss, torch.zeros_like(ss, dtype=torch.long), 0.5)
        d = torch.cat([bb[k], ss[k, None]], 1).cpu().numpy()                 # bbox2result
        d[:, [0, 2]] += m[0]['tile_offset'][0]
        d[:, [1, 3]] += m[0]['tile_offset'][1]
        all_b.append(d)
        all_l.append(torch.zeros(len(d), dtype=torch.long))
    b = torch.from_numpy(np.concatenate(all_b)).cuda()
    lab = torch.cat(all_l).cuda()
    keep = torchvision.ops.batched_nms(b[:, :4], b[:, 4], lab, 0.5)
    return b[keep].cpu().numpy()


def timed(fn, runs):
    out = []
    for _ in range(runs):
        torch.cuda.synchronize()
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t) * 1e3)
    return out


def fmt(ts):
    return f'{np.median(ts):.2f} ms ({min(ts):.2f} - {max(ts):.2f})'


def nms_rows(n, g):
    xy = torch.rand(n, 2, generator=g) * torch.tensor([1920., 1080.])
    wh = 6 + torch.rand(n, 2, generator=g) * 30
    return torch.cat([xy, xy + wh, torch.rand(n, 1, generator=g)], 1).cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=20)
    ap.add_argument('--logits', choices=['realistic', 'scaled'], default='realistic')
    ap.add_argument('--profile', default=None)
    a = ap.parse_args()
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    rpn, roi, feats, metas, rpn_cfg, test = build(a.logits == 'scaled')
    with torch.no_grad():
        ours = lambda: tile_aug_test(rpn, roi, feats, copy.deepcopy(metas), test)
        ref = lambda: reference_ops(rpn, roi, feats, metas, rpn_cfg, test)
        r = ours()
        n_ref = len(ref())
        print(f'card: {card}; logits {a.logits}: tile_aug_test {r[0][0].shape[0]} detections, reference ops {n_ref}')
        if a.profile:
            os.makedirs(a.profile, exist_ok=True)
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as prof:
                ours()
                torch.cuda.synchronize()
            table = prof.key_averages().table(sort_by='cuda_time_total', row_limit=30)
            open(os.path.join(a.profile, f'tile_test_profile_{a.logits}.txt'), 'w').write(table)
            print(table)
            return
        g = torch.Generator().manual_seed(1)
        rows = {n: nms_rows(n, g) for n in (12000, 65536)}
        zero = {n: torch.zeros(n, dtype=torch.long, device='cuda') for n in rows}
        arms = {'tile_aug_test': ours, 'reference ops': ref}
        for n, x in rows.items():
            x3, lab = x[None].contiguous(), zero[n].int()[None].contiguous()
            arms[f'ptb_batched_nms {n}'] = lambda x3=x3, lab=lab: ops.batched_nms(x3, x3[..., 4], lab, None, 0.5)
            arms[f'torchvision batched_nms {n}'] = lambda x=x, z=zero[n]: torchvision.ops.batched_nms(x[:, :4], x[:, 4], z, 0.5)
        for f in arms.values():
            timed(f, 3)
        res = {k: [] for k in arms}
        for _ in range(a.runs):                 # alternate the arms
            for k, f in arms.items():
                res[k] += timed(f, 1)
        for k, ts in res.items():
            print(f'{k:32s} {fmt(ts)}')


if __name__ == '__main__':
    main()
