"""Pins oracle/roi_head.py against the REAL reference and writes tests/golden/roi_head_*.npz.  (test infrastructure)

Run in the build container only (needs /root/reference):   python -m oracle.make_golden_roi_head
The unmodified reference mmdet package is imported through oracle/_mmcv_stub.py with mmcv.ops.RoIAlign bound to oracle.roi_head.RoIAlign
(the restatement of mmcv's CPU kernel, pinned to torchvision).  For every case of oracle.roi_head.CASES a reference StandardRoIHead is
built with the case's seeded weights; forward_train runs from torch.manual_seed(case seed) and is back-propagated, simple_test runs on
the same inputs; the oracle then runs from the same seed and their agreement is ASSERTED: sampled sets, rois, labels and weights equal,
targets within 1e-6, cls_score / bbox_pred, losses and acc within 1e-6, every gradient within 1e-5, the generator state after the call
equal, detections equal.  Stored (small: the inputs are regenerated from the seeds): the sampled sets, labels, targets, losses, acc, the
generator state, gradient samples and sums, the detections, and the reference classes' constructor keywords and state_dict names / shapes.
"""
import inspect
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import roi_head as orh  # noqa: E402
from oracle import _mmcv_stub as stub  # noqa: E402
from oracle.make_golden import GOLD, eq, sub  # noqa: E402


def cfgdict(d):
    return stub.CfgDict({k: cfgdict(v) if isinstance(v, dict) else v for k, v in d.items()})


def golden_case(HEADS, name):
    c = orh.CASES[name]
    inp = orh.case_inputs(name)
    head = HEADS.build(dict(type='StandardRoIHead', **orh.head_kwargs(name), train_cfg=cfgdict(c['train']), test_cfg=cfgdict(c['test'])))
    head.bbox_head.load_state_dict(inp['weights'], strict=True)
    sampled = []
    real_sample = head.bbox_sampler.sample
    head.bbox_sampler.sample = lambda *a, **k: sampled.append(real_sample(*a, **k)) or sampled[-1]
    feats = [f.clone().requires_grad_(True) for f in inp['feats']]
    torch.manual_seed(c['seed'])
    losses = head.forward_train(feats, inp['img_metas'], [p.clone() for p in inp['proposals']], inp['gt_bboxes'], inp['gt_labels'])
    state = torch.get_rng_state()
    (losses['loss_cls'] + losses['loss_bbox']).backward()
    # the oracle from the same seed and weights
    of = [f.clone().requires_grad_(True) for f in inp['feats']]
    w = {k: v.clone().requires_grad_(True) for k, v in inp['weights'].items()}
    torch.manual_seed(c['seed'])
    ol, tg = orh.forward_train(inp, name, feats=of, w=w)
    assert torch.equal(torch.get_rng_state(), state), f'{name}: generator state'
    (ol['loss_cls'] + ol['loss_bbox']).backward()
    out = dict(seed=np.int64(c['seed']), rng_state=state.numpy())
    for b, s in enumerate(sampled):
        eq(tg['samples'][b][2], s.pos_inds, f'{name} pos {b}')
        eq(tg['samples'][b][3], s.neg_inds, f'{name} neg {b}')
        out[f'pos_inds{b}'], out[f'neg_inds{b}'] = s.pos_inds.numpy(), s.neg_inds.numpy()
    from mmdet.core import bbox2roi
    rois = bbox2roi([s.bboxes for s in sampled])
    ref_tg = head.bbox_head.get_targets(sampled, inp['gt_bboxes'], inp['gt_labels'], head.train_cfg)
    eq(tg['rois'], rois, f'{name} rois')
    for k, key in enumerate(('labels', 'label_weights', 'bbox_targets', 'bbox_weights')):
        eq(tg[key], ref_tg[k], f'{name} {key}', exact=key != 'bbox_targets')
        out[key] = ref_tg[k].numpy()
    out['rois'] = rois.numpy()
    for k in ('loss_cls', 'loss_bbox', 'acc'):
        eq(ol[k].detach(), losses[k].detach(), f'{name} {k}', exact=False)
        out[k] = losses[k].detach().numpy()
    assert feats[-1].grad is None and of[-1].grad is None            # x[:num_inputs]: the fifth level is not read
    for l in range(len(orh.STRIDES)):
        eq(of[l].grad, feats[l].grad, f'{name} grad feat{l}', exact=False, tol=1e-5)
        out[f'grad_feat{l}_sub'], out[f'grad_feat{l}_sum'], out[f'grad_feat{l}_abssum'] = sub(feats[l].grad, 97)
    for k, p in head.bbox_head.named_parameters():
        eq(w[k].grad, p.grad, f'{name} grad {k}', exact=False, tol=1e-5)
        out[f'grad/{k}_sub'], out[f'grad/{k}_sum'], out[f'grad/{k}_abssum'] = sub(p.grad, 41)
    # simple_test, the reference's batched path and the oracle's
    with torch.no_grad():
        res = head.simple_test(tuple(inp['feats']), [p.clone() for p in inp['proposals']], inp['img_metas'])
        od, olab = orh.simple_test(inp, name)
    C = c['head']['num_classes']
    for b in range(len(res)):
        mine = [od[b][olab[b] == k].numpy() for k in range(C)]
        for k in range(C):
            assert mine[k].shape[0] == res[b][k].shape[0], f'{name} dets img {b} class {k}: count'
            if mine[k].shape[0]:
                eq(torch.from_numpy(mine[k]), torch.from_numpy(res[b][k]), f'{name} dets img {b} class {k}', exact=False)
        out[f'dets{b}'] = od[b].numpy()
        out[f'det_labels{b}'] = olab[b].numpy().astype(np.int16)
    sd = head.state_dict()
    out['state_keys'] = np.array(list(sd))                  # in registration order: optimizer state is indexed by it
    out['state_shapes'] = np.array([list(sd[k].shape) + [-1] * (2 - sd[k].dim()) for k in sd], np.int64)
    path = os.path.join(GOLD, f'roi_head_{name}.npz')
    np.savez_compressed(path, **out)
    print(f'[golden] {path}: {os.path.getsize(path) / 1024:.0f} KiB, rois {rois.shape[0]}, dets {[len(d) for d in od]}')


def golden_ctor():
    """the reference classes' constructor keywords"""
    from mmdet.models.roi_heads import StandardRoIHead, SingleRoIExtractor
    from mmdet.models.roi_heads.base_roi_head import BaseRoIHead
    from mmdet.models.roi_heads.bbox_heads import Shared2FCBBoxHead
    from mmdet.models.roi_heads.bbox_heads.bbox_head import BBoxHead
    from mmdet.models.roi_heads.bbox_heads.convfc_bbox_head import ConvFCBBoxHead
    names = lambda f, drop=(): [p for p in inspect.signature(f).parameters if p not in ('self', 'args', 'kwargs') + tuple(drop)]
    fixed = ('num_shared_convs', 'num_shared_fcs', 'num_cls_convs', 'num_cls_fcs', 'num_reg_convs', 'num_reg_fcs')
    out = dict(roi_head=np.array(names(BaseRoIHead.__init__)), extractor=np.array(names(SingleRoIExtractor.__init__)),
               bbox_head=np.array(names(Shared2FCBBoxHead.__init__) + names(ConvFCBBoxHead.__init__, fixed + ('init_cfg',))
                                  + names(BBoxHead.__init__)))
    assert StandardRoIHead.__init__ is BaseRoIHead.__init__
    path = os.path.join(GOLD, 'roi_head_ctor.npz')
    np.savez_compressed(path, **out)
    print(f'[golden] {path}')


def main():
    torch.set_num_threads(1)             # the CPU sums (gradients) reduce in a thread-count-dependent order: one thread reproduces them
    stub.KNOWN['mmcv.ops']['RoIAlign'] = orh.RoIAlign
    stub.Registry.__contains__ = lambda self, key: self.get(key) is not None      # mmdet's build_linear_layer tests membership
    HEADS = stub.load_reference()
    for name in orh.CASES:
        golden_case(HEADS, name)
    golden_ctor()


if __name__ == '__main__':
    main()
