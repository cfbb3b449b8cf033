"""Pins oracle/rpn_loss.py against the REAL reference and writes tests/golden/rpn_loss_*.npz.  (test infrastructure)

Run in the build container only (needs /root/reference):   python -m oracle.make_golden_rpn_loss
The unmodified reference mmdet package is imported through oracle/_mmcv_stub.py, an RPNHead is built for every case of
oracle.rpn_loss.CASES with the case's seeded conv weights, and RPNHead.loss runs from torch.manual_seed(case seed) on the case's features;
the oracle then runs from the same seed, and their agreement is ASSERTED: sampled sets, labels and weights equal, bbox targets, losses and
gradients within 1e-6, the CPU generator state after the call equal.  Stored: the sampled sets, the real head's targets
(AnchorHead.get_targets run again from the same seed, every entry asserted against the oracle's, in images_to_levels layout), the
per-level losses, the gradients of the output maps (strided samples + sums) and of the three convs, the generator state after the call, and
the reference head's constructor parameters and state_dict names / shapes.  rpn_loss_roi_sampler.npz: RandomSampler(num=512,
pos_fraction=0.25, add_gt_as_proposals=True) alone on an R-CNN-stage assignment.
"""
import inspect
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import rpn_loss as orl  # noqa: E402
from oracle._mmcv_stub import load_reference, CfgDict  # noqa: E402
from oracle.make_golden import GOLD, eq, sub  # noqa: E402


def cfgdict(d):
    return CfgDict({k: cfgdict(v) if isinstance(v, dict) else v for k, v in d.items()})


def golden_case(HEADS, name):
    c = orl.CASES[name]
    inp = orl.case_inputs(name)
    head = HEADS.build(dict(type='RPNHead', **orl.head_kwargs(name), train_cfg=cfgdict(c['train'])))
    head.load_state_dict(inp['weights'], strict=True)
    sampled = []
    real_sample = head.sampler.sample
    head.sampler.sample = lambda *a, **k: sampled.append(real_sample(*a, **k)) or sampled[-1]
    feats = [f.clone().requires_grad_(True) for f in inp['feats']]
    cls, reg = head(feats)
    for t in cls + reg:
        t.retain_grad()
    torch.manual_seed(c['seed'])
    losses = head.loss(cls, reg, inp['gt_bboxes'], inp['img_metas'], gt_bboxes_ignore=inp['gt_bboxes_ignore'])
    state = torch.get_rng_state()
    sum(sum(v) for v in losses.values()).backward()
    # the oracle from the same seed and weights
    w = {k: v.clone().requires_grad_(True) for k, v in inp['weights'].items()}
    ocls, oreg = orl.forward(inp['feats'], w)
    for t in ocls + oreg:
        t.retain_grad()
    torch.manual_seed(c['seed'])
    ol, tg = orl.loss(ocls, oreg, inp['gt_bboxes'], inp['img_metas'], inp['gt_bboxes_ignore'], orl.head_kwargs(name), c['train'])
    assert torch.equal(torch.get_rng_state(), state), f'{name}: generator state'
    sum(sum(v) for v in ol.values()).backward()
    out = dict(seed=np.int64(c['seed']), rng_state=state.numpy(), num_total_samples=np.int64(tg['num_total_samples']))
    for b, s in enumerate(sampled):
        eq(tg['pos_inds'][b], s.pos_inds, f'{name} pos {b}')
        eq(tg['neg_inds'][b], s.neg_inds, f'{name} neg {b}')
        out[f'pos_inds{b}'], out[f'neg_inds{b}'] = s.pos_inds.numpy(), s.neg_inds.numpy()
    # the real head's targets (AnchorHead.get_targets from the same seed, the same draws), every entry against the oracle's
    torch.manual_seed(c['seed'])
    anchor_list, valid_flag_list = head.get_anchors([t.shape[-2:] for t in cls], inp['img_metas'], device='cpu')
    ref_tg = head.get_targets(anchor_list, valid_flag_list, inp['gt_bboxes'], inp['img_metas'],
                              gt_bboxes_ignore_list=inp['gt_bboxes_ignore'], gt_labels_list=None, label_channels=1)
    assert torch.equal(torch.get_rng_state(), state), f'{name}: generator state after get_targets'
    assert ref_tg[4] + ref_tg[5] == tg['num_total_samples']
    for l, (lab, lw, bt, bw) in enumerate(tg['levels']):
        rlab, rlw, rbt, rbw = (ref_tg[k][l] for k in range(4))
        eq(lab, rlab, f'{name} labels{l}')
        eq(lw, rlw, f'{name} label_weights{l}')
        eq(bw, rbw, f'{name} bbox_weights{l}')
        eq(bt, rbt, f'{name} bbox_targets{l}', exact=False)
        out[f'labels{l}'], out[f'label_weights{l}'] = rlab.numpy().astype(np.int8), rlw.numpy()
        out[f'bbox_targets{l}'], out[f'bbox_weights{l}'] = rbt.numpy(), rbw.numpy().astype(np.int8)
        for key, mine, ref in (('loss_cls', ol['loss_rpn_cls'][l], losses['loss_rpn_cls'][l]),
                               ('loss_bbox', ol['loss_rpn_bbox'][l], losses['loss_rpn_bbox'][l])):
            eq(mine.detach(), ref.detach(), f'{name} {key}{l}', exact=False)
            out[f'{key}{l}'] = ref.detach().numpy()
        for key, mine, ref in (('grad_cls', ocls[l].grad, cls[l].grad), ('grad_reg', oreg[l].grad, reg[l].grad)):
            eq(mine, ref, f'{name} {key}{l}', exact=False)
            out[f'{key}{l}_sub'], out[f'{key}{l}_sum'], out[f'{key}{l}_abssum'] = sub(ref, 7)
    for k, p in head.named_parameters():
        eq(w[k].grad, p.grad, f'{name} grad {k}', exact=False)
        out[f'grad/{k}'] = p.grad.numpy()
    sd = head.state_dict()
    out['state_keys'] = np.array(sorted(sd))
    out['state_shapes'] = np.array([list(sd[k].shape) + [-1] * (4 - sd[k].dim()) for k in sorted(sd)], np.int64)
    from mmdet.models.dense_heads.anchor_head import AnchorHead
    from mmdet.models.dense_heads.rpn_head import RPNHead
    params = [p for p in inspect.signature(RPNHead.__init__).parameters if p not in ('self', 'kwargs')]
    params += [p for p in inspect.signature(AnchorHead.__init__).parameters if p not in ('self', 'num_classes', 'in_channels', 'init_cfg')]
    out['ctor_params'] = np.array(params)
    path = os.path.join(GOLD, f'rpn_loss_{name}.npz')
    np.savez_compressed(path, **out)
    print(f'[golden] {path}: {os.path.getsize(path) / 1024:.0f} KiB, num_total_samples {tg["num_total_samples"]}, '
          f'pos {[len(p) for p in tg["pos_inds"]]}, neg {[len(n) for n in tg["neg_inds"]]}')


def golden_roi_sampler():
    from mmdet.core.bbox.samplers import RandomSampler
    from mmdet.core.bbox.assigners.assign_result import AssignResult
    anchors, gts, labels, gt_inds, max_ov, lab = orl.roi_sampler_inputs()
    s = RandomSampler(**orl.ROI_SAMPLER)
    torch.manual_seed(21)
    r = s.sample(AssignResult(gts.shape[0], gt_inds.clone(), max_ov.clone(), lab.clone()), anchors, gts, labels)
    out = dict(pos_inds=r.pos_inds.numpy(), neg_inds=r.neg_inds.numpy(), pos_is_gt=r.pos_is_gt.numpy(),
               pos_assigned_gt_inds=r.pos_assigned_gt_inds.numpy(), pos_gt_labels=r.pos_gt_labels.numpy(), rng_state=torch.get_rng_state().numpy())
    # the oracle's sampler on the same assignment with the GTs prepended
    torch.manual_seed(21)
    full = torch.cat([torch.arange(1, gts.shape[0] + 1), gt_inds])
    pos, neg = orl.random_sample(full, orl.ROI_SAMPLER['num'], orl.ROI_SAMPLER['pos_fraction'])
    eq(pos, r.pos_inds, 'roi pos')
    eq(neg, r.neg_inds, 'roi neg')
    assert torch.equal(torch.get_rng_state(), torch.from_numpy(out['rng_state']))
    path = os.path.join(GOLD, 'rpn_loss_roi_sampler.npz')
    np.savez_compressed(path, **out)
    print(f'[golden] {path}: pos {len(pos)}, neg {len(neg)}')


def main():
    torch.set_num_threads(os.cpu_count())
    HEADS = load_reference()
    for name in orl.CASES:
        golden_case(HEADS, name)
    golden_roi_sampler()


if __name__ == '__main__':
    main()
