"""FCOSHead on the TinyPerson shapes (1 class, strides 8-128, 256 channels, 640 x 512 tiles): three workloads, each timed against the
reference's op sequence on the same GPU (oracle/fcos.py on CUDA tensors: cuDNN fp32 convs with TF32 off, the reference's torch loss with
its nonzero and host reads, torchvision batched_nms for mmcv's), the two arms alternating in one process; median (min - max) of --runs.
  train       16 tiles, 5 levels, 24 GTs per tile: forward + loss + backward
  simple_test 16 tiles: forward + get_bboxes
  aug_test    one 1920 x 1080 image in 12 tiles (tile_offset), aug_test_bboxes
--profile OUT_DIR splits the device time of one training step and one aug_test between towers, output convs, targets, losses, decode
and NMS (torch.profiler, a run of its own).
    python tools/bench_fcos.py [--runs 20] [--profile OUT_DIR]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torchvision

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import fcos as ofc  # noqa: E402
from pointtinybenchmark_b200.fcos_head import FCOSHead  # noqa: E402

B_TRAIN, TH, TW = 16, 512, 640


def setup():
    g = torch.Generator().manual_seed(0)
    head = FCOSHead(**ofc.head_kwargs('tinyperson')).cuda()
    w = {k: v.cuda() for k, v in ofc.weights(g, 1).items()}
    head.load_state_dict(w, strict=True)
    sizes = ofc.featmap_sizes((TH, TW), ofc.TINY['strides'])
    feats = [torch.randn(B_TRAIN, 256, h, wd, generator=g).cuda() for h, wd in sizes]
    gts, gls = [], []
    for _ in range(B_TRAIN):
        b, l = ofc.gt_boxes(g, 24, (TH, TW))
        gts.append(b.cuda()); gls.append(l.cuda())
    metas = [dict(img_shape=(TH, TW, 3), pad_shape=(TH, TW, 3), scale_factor=np.ones(4, np.float32), flip=False, flip_direction=None)
             for _ in range(B_TRAIN)]
    tiles = [[f[:1].clone() for f in feats] for _ in ofc.TILE_OFFSETS]
    tmetas = [[dict(metas[0], ori_shape=(1080, 1920, 3), tile_offset=o)] for o in ofc.TILE_OFFSETS]
    return head, w, feats, gts, gls, metas, tiles, tmetas


def ref_nms(boxes, scores, factors, cfg):
    valid = scores > cfg['score_thr']
    inds = valid.nonzero()
    b, s, l = boxes[inds[:, 0]], (scores * factors[:, None])[valid], inds[:, 1]
    keep = torchvision.ops.batched_nms(b, s, l, cfg['nms']['iou_threshold'])[:cfg['max_per_img']]
    return torch.cat([b[keep], s[keep, None]], -1), l[keep]


def ours_train(head, feats, gts, gls, metas):
    head.zero_grad(set_to_none=True)
    losses = head.loss(*head(feats), gts, gls, metas)
    sum(losses.values()).backward()


def ref_train(w, feats, gts, gls):
    ws = {k: v.detach().requires_grad_(True) for k, v in w.items()}
    cfg = dict(ofc.TINY, stacked_convs=4)
    losses, _ = ofc.loss(*ofc.forward(feats, ws, cfg, True), gts, gls, cfg)
    sum(losses.values()).backward()


def ours_test(head, feats, metas):
    with torch.no_grad():
        return head.simple_test(feats, metas)


def ref_test(w, feats, metas):
    cfg = dict(ofc.TINY, stacked_convs=4)
    with torch.no_grad():
        bb, sc, kk, _ = ofc.decode(*ofc.forward(feats, w, cfg, False), metas, cfg, ofc.TINY_TEST)
        return [ref_nms(bb[b], sc[b], kk[b], ofc.TINY_TEST) for b in range(bb.shape[0])]


def ours_aug(head, tiles, tmetas):
    with torch.no_grad():
        return head.aug_test(tiles, tmetas)


def ref_aug(w, tiles, tmetas):
    cfg = dict(ofc.TINY, stacked_convs=4)
    boxes, scores, facs = [], [], []
    with torch.no_grad():
        for x, m in zip(tiles, tmetas):
            bb, sc, kk, _ = ofc.decode(*ofc.forward(x, w, cfg, False), m, cfg, ofc.TINY_TEST)
            boxes.append(bb[0] + bb.new_tensor(m[0]['tile_offset']).repeat(2))      # bbox_mapping_back of an unflipped, unscaled tile
            scores.append(sc[0]); facs.append(kk[0])
        d, l = ref_nms(torch.cat(boxes), torch.cat(scores), torch.cat(facs), ofc.TINY_TEST)
        d = d.clone()
        d[:, :4] *= d.new_tensor(tmetas[0][0]['scale_factor'])
        return d, l


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def profile(out_dir, head, feats, gts, gls, metas, tiles, tmetas):
    from torch.profiler import ProfilerActivity, profile as prof
    os.makedirs(out_dir, exist_ok=True)
    groups = [('output convs (wgmma)', ('conv_tc_kernel<true, 16',)),
              ('towers', ('conv_tc_kernel', 'conv3x3', 'wgrad_tc', 'wgrad_reduce', 'gn_', 'split_f16', 'amax_abs', 'col_sum')),
              ('output convs (cuDNN)', ('xmma', 'cudnn', 'conv2d_precomputed', 'gemvx', 'winograd', 'implicit_convolve')),
              ('targets', ('fcos_targets',)), ('losses', ('loss_sum_kernel',)), ('decode', ('fcos_key', 'fcos_gather', 'p2p_select')),
              ('nms', ('nms', 'map_back'))]
    res = {}
    for name, fn in (('train', lambda: ours_train(head, feats, gts, gls, metas)), ('aug_test', lambda: ours_aug(head, tiles, tmetas))):
        fn(); torch.cuda.synchronize()
        with prof(activities=[ProfilerActivity.CUDA]) as p:
            fn(); torch.cuda.synchronize()
        split = {}
        for e in p.key_averages():
            if e.device_type.name != 'CUDA' or e.self_device_time_total <= 0:
                continue
            key = next((k for k, pats in groups if any(s in e.key for s in pats)), 'torch glue (flatten, exp, cat, fill)')
            split[key] = split.get(key, 0.0) + e.self_device_time_total / 1e3
        res[name] = {k: round(v, 3) for k, v in sorted(split.items(), key=lambda kv: -kv[1])}
        with open(os.path.join(out_dir, f'fcos_{name}_kernels.txt'), 'w') as f:
            f.write(p.key_averages().table(sort_by='self_cuda_time_total', row_limit=40))
    print(json.dumps(dict(profile_ms=res)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=20)
    ap.add_argument('--profile', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_fcos needs a CUDA device')
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    head, w, feats, gts, gls, metas, tiles, tmetas = setup()
    if a.profile:
        profile(a.profile, head, feats, gts, gls, metas, tiles, tmetas)
        return
    work = {'train': (lambda: ours_train(head.train(), feats, gts, gls, metas), lambda: ref_train(w, feats, gts, gls)),
            'simple_test': (lambda: ours_test(head.eval(), feats, metas), lambda: ref_test(w, feats, metas)),
            'aug_test': (lambda: ours_aug(head.eval(), tiles, tmetas), lambda: ref_aug(w, tiles, tmetas))}
    info = gpu_info()
    out = dict(gpu=info, runs=a.runs)
    for name, (ours, ref) in work.items():
        for _ in range(3):
            ours(); ref()
        t_o, t_r = [], []
        for _ in range(a.runs):
            t_o.append(timed(ours)); t_r.append(timed(ref))
        st = lambda t: dict(median=round(float(np.median(t)), 2), min=round(min(t), 2), max=round(max(t), 2))
        out[name] = dict(fcos_head_ms=st(t_o), reference_ops_ms=st(t_r))
    d, l = ours_aug(head.eval(), tiles, tmetas)[0]
    rd, rl = ref_aug(w, tiles, tmetas)
    out['aug_test_detections'] = [int(d.shape[0]), int(rd.shape[0])]
    print(json.dumps(out))


if __name__ == '__main__':
    main()
