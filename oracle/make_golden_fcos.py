"""Pins oracle/fcos.py against the REAL reference FCOSHead and writes tests/golden/fcos_*.npz.  (test infrastructure)

Run in the build container only (needs /root/reference):   python -m oracle.make_golden_fcos
The unmodified reference mmdet package is imported through oracle/_mmcv_stub.py, with mmcv.cnn.Scale restated (a `scale` parameter,
forward x * scale).  For every case of oracle.fcos.CASES the reference head is built with the case's seeded weights and runs forward (the
cases with towers), loss and backward, get_targets and get_bboxes; the oracle runs on the same inputs and is ASSERTED equal: labels, bbox
targets, top-k rows and kept detections bit-exact, losses and gradients within 1e-6.  The tile cases run the reference's aug_test_bboxes
with `forward` replaced by the seeded per-aug maps.  Stored: the reference's output maps, targets, losses, gradients (large ones as strided
samples + sums), detections, and for tinyperson / coco80 the constructor parameters and state_dict names and shapes."""
import inspect
import os
import sys

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import fcos as ofc  # noqa: E402
from oracle import _mmcv_stub as stub  # noqa: E402
from oracle.make_golden import GOLD, eq, sub  # noqa: E402


class Scale(nn.Module):
    """mmcv.cnn.Scale restated"""

    def __init__(self, scale=1.0):
        super().__init__()
        self.scale = nn.Parameter(torch.tensor(scale, dtype=torch.float))

    def forward(self, x):
        return x * self.scale


def load():
    stub.KNOWN['mmcv.cnn']['Scale'] = Scale
    HEADS = stub.load_reference()
    sys.modules[HEADS.get('FCOSHead').__module__].Scale = Scale
    return HEADS


def cfgdict(d):
    return stub.CfgDict({k: cfgdict(v) if isinstance(v, dict) else v for k, v in d.items()})


def build(HEADS, kw):
    kw = dict(kw)
    kw['test_cfg'] = cfgdict(kw['test_cfg'])
    return HEADS.build(dict(type='FCOSHead', **kw))


def store_maps(out, key, maps):
    for n, ts in zip(('cls', 'reg', 'ctr'), maps):
        for l, t in enumerate(ts):
            out[f'{key}_{n}{l}'] = t.detach().numpy()


def golden_case(HEADS, name):
    c = ofc.CASES[name]
    inp = ofc.case_inputs(name)
    kw = ofc.head_kwargs(name)
    cfg, test_cfg = dict(c['head']), c['test']
    cfg['stacked_convs'] = 4
    head = build(HEADS, kw)
    head.load_state_dict(inp['weights'], strict=True)
    out = {}
    gts, gls, metas = inp['gt_bboxes'], inp['gt_labels'], inp['img_metas']
    w = {k: v.clone().requires_grad_(True) for k, v in inp['weights'].items()}
    if c['towers']:
        head.train()
        maps = head([f.clone() for f in inp['feats']])
        omaps = ofc.forward(inp['feats'], w, cfg, training=True)
    else:
        maps = tuple([t.clone().requires_grad_(True) for t in ts] for ts in inp['maps'])
        omaps = tuple([t.clone().requires_grad_(True) for t in ts] for ts in inp['maps'])
    for ts in maps + omaps:
        for t in ts:
            t.retain_grad()
    for a, b in zip(sum(map(list, maps), []), sum(map(list, omaps), [])):
        eq(b.detach(), a.detach(), f'{name} forward', exact=False)
    if c['towers']:
        store_maps(out, 'train', maps)
    losses = head.loss(*maps, gts, gls, metas)
    ol, tg = ofc.loss(*omaps, gts, gls, cfg)
    for k in ('loss_cls', 'loss_bbox', 'loss_centerness'):
        eq(ol[k].detach(), losses[k].detach(), f'{name} {k}', exact=False)
        out[k] = losses[k].detach().numpy()
    sum(losses.values()).backward()
    sum(ol.values()).backward()
    for n, ts, os_ in zip(('cls', 'reg', 'ctr'), maps, omaps):
        for l, (a, b) in enumerate(zip(ts, os_)):
            if a.grad is None:
                assert b.grad is None or not b.grad.any()
                continue
            eq(b.grad, a.grad, f'{name} grad {n}{l}', exact=False)
            if a.grad.numel() > 65536:
                out[f'grad_{n}{l}_sub'], out[f'grad_{n}{l}_sum'], out[f'grad_{n}{l}_abssum'] = sub(a.grad, 7)
            else:
                out[f'grad_{n}{l}'] = a.grad.numpy()
    if c['towers']:
        for k, p in head.named_parameters():
            eq(w[k].grad, p.grad, f'{name} grad {k}', exact=False)
            if p.numel() > 4096:
                out[f'pgrad/{k}_sub'], out[f'pgrad/{k}_sum'], out[f'pgrad/{k}_abssum'] = sub(p.grad, 97)
            else:
                out[f'pgrad/{k}'] = p.grad.numpy()
    pts = head.get_points([t.shape[-2:] for t in maps[0]], torch.float32, 'cpu')
    rl, rt = head.get_targets(pts, gts, gls)
    for l in range(len(rl)):
        eq(tg['labels'][l], rl[l], f'{name} labels{l}')
        eq(tg['bbox_targets'][l], rt[l], f'{name} bbox_targets{l}')
        out[f'labels{l}'] = rl[l].numpy().astype(np.int16)
        out[f'bbox_targets{l}'] = rt[l].numpy()
    # test
    head.eval()
    with torch.no_grad():
        emaps = head([f.clone() for f in inp['feats']]) if c['towers'] else tuple([t.detach() for t in ts] for ts in inp['maps'])
        if c['towers']:
            oe = ofc.forward(inp['feats'], inp['weights'], cfg, training=False)
            for a, b in zip(sum(map(list, emaps), []), sum(map(list, oe), [])):
                eq(b, a, f'{name} eval forward', exact=False)
            store_maps(out, 'eval', emaps)
        rescale = c.get('rescale', False)
        raw = head.get_bboxes(*emaps, metas, rescale=rescale, with_nms=False)
        res = head.get_bboxes(*emaps, metas, rescale=rescale)
        # the oracle decodes from the reference's own maps: equal rows before the NMS, equal detections after it
        bb, sc, kk, tk = ofc.decode(*emaps, metas, cfg, test_cfg, rescale)
        ores, _ = ofc.get_bboxes(*emaps, metas, cfg, test_cfg, rescale)
    for b in range(len(metas)):
        eq(bb[b], raw[b][0], f'{name} boxes {b}')
        eq(sc[b], raw[b][1][:, :-1], f'{name} scores {b}')
        eq(kk[b], raw[b][2], f'{name} centerness {b}')
        eq(ores[b][0], res[b][0], f'{name} dets {b}')
        eq(ores[b][1], res[b][1], f'{name} det labels {b}')
        out[f'dets{b}'], out[f'det_labels{b}'] = res[b][0].numpy(), res[b][1].numpy().astype(np.int16)
    for l, t in enumerate(tk):
        if t is not None:
            out[f'topk{l}'] = t.numpy().astype(np.int32)
    if name in ('tinyperson', 'coco80'):
        sd = head.state_dict()
        out['state_keys'] = np.array(sorted(sd))
        out['state_shapes'] = np.array([list(sd[k].shape) + [-1] * (4 - sd[k].dim()) for k in sorted(sd)], np.int64)
        FCOSHead = HEADS.get('FCOSHead')
        AnchorFreeHead = FCOSHead.__mro__[1]
        params = [p for p in inspect.signature(FCOSHead.__init__).parameters if p not in ('self', 'kwargs')]
        params += [p for p in inspect.signature(AnchorFreeHead.__init__).parameters if p not in ('self', 'num_classes', 'in_channels',
                                                                                                  'loss_cls', 'loss_bbox', 'norm_cfg', 'init_cfg')]
        out['ctor_params'] = np.array(params)
    path = os.path.join(GOLD, f'fcos_{name}.npz')
    np.savez_compressed(path, **out)
    npos = sum(int(((l >= 0) & (l < cfg['num_classes'])).sum()) for l in rl)
    print(f'[golden] {path}: {os.path.getsize(path) / 1024:.0f} KiB, {npos} positives, dets {[len(r[0]) for r in res]}')


def golden_tiles(HEADS, name):
    augs = ofc.tile_case(name)
    kw = ofc.head_kwargs('tinyperson')
    head = build(HEADS, kw)
    head.eval()
    maps = [ofc.aug_maps(a) for a in augs]
    calls = iter(maps)
    head.forward = lambda x: next(calls)              # the reference's aug_test_bboxes on the seeded per-aug maps
    metas = [[a['meta']] for a in augs]
    feats = [[torch.zeros(1, 1, h, w) for h, w in a['sizes']] for a in augs]
    out = {}
    for rescale in (False, True):
        calls = iter(maps)
        head.forward = lambda x: next(calls)
        with torch.no_grad():
            d, l = head.aug_test_bboxes(feats, metas, rescale=rescale)[0]
            od, ol, rows = ofc.aug_test_bboxes(maps, metas, ofc.TINY, ofc.TINY_TEST, rescale=rescale)
        eq(od, d, f'{name} dets rescale={rescale}')
        eq(ol, l, f'{name} labels rescale={rescale}')
        out[f'dets_rescale{int(rescale)}'], out[f'labels_rescale{int(rescale)}'] = d.numpy(), l.numpy().astype(np.int16)
    out['rows'] = np.int64(rows)
    out['seeds'] = np.array([a['seed'] for a in augs], np.int64)
    path = os.path.join(GOLD, f'fcos_{name}.npz')
    np.savez_compressed(path, **out)
    print(f'[golden] {path}: {os.path.getsize(path) / 1024:.0f} KiB, {rows} rows at the merge, {len(out["dets_rescale0"])} detections')


def main():
    torch.set_num_threads(os.cpu_count())
    HEADS = load()
    names = sys.argv[1:] or list(ofc.CASES) + ['tiles', 'flip_scale']
    for name in names:
        if name in ofc.CASES:
            golden_case(HEADS, name)
        else:
            golden_tiles(HEADS, name)


if __name__ == '__main__':
    main()
