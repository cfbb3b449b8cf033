"""Pins the oracle's MILLoss(loss_type='binary_cross_entropy') and AllPosLoss (oracle/cpr_loss_types.py) against the REAL reference and writes
tests/golden/cpr_lite_loss_<case>.npz.  (test infrastructure)

Run in the build container only (needs /root/reference):   python -m oracle.make_golden_cpr_loss_types
Same procedure as oracle/make_golden.py::golden_cpr_variant: the unmodified reference CPRHead is built through oracle/_mmcv_stub.py with
the case's `loss_mil` (and variant) kwargs, reference and oracle run the loss and its backward on the same seeded inputs, their equality
is ASSERTED (1e-6), then the reference's losses and gradients are stored.  The inputs are CPR-lite plus one GT whose whole ring bag lies
outside pad_shape (a fully invalid bag: prob = 0, which BCE scores 100 at the label column); the variant case also has a zero-weight
bag (gt_weights).  The inputs are asserted free of near-ties that would make bag_acc fragile: for every bag (MIL) or bag sample
(AllPos) the label's probability is at least 1e-5 away from the largest other class's, so a top-1 hit is decided the same way by any
computation accurate to 1e-5.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import cpr as ocpr, cpr_loss_types as olt, synth  # noqa: E402
from oracle._mmcv_stub import load_reference  # noqa: E402
from oracle.make_golden import GOLD, eq, ref_cpr_cfg, sub  # noqa: E402

SEED = 1235
TIE = 1e-5

# case -> (reference ctor overrides, oracle cfg overrides, with gt_weights)
LOSS_TYPE_CASES = {
    'mil_bce': (dict(loss_mil=dict(type='MILLoss', binary_ins=False, loss_weight=0.25, loss_type='binary_cross_entropy')),
                dict(mil_loss_type='binary_cross_entropy'), False),
    'allpos_gfocal': (dict(loss_mil=dict(type='AllPosLoss', binary_ins=False, loss_weight=0.25, loss_type='gfocal_loss')),
                      dict(loss_mil='AllPosLoss', mil_loss_type='gfocal_loss'), False),
    'allpos_bce': (dict(loss_mil=dict(type='AllPosLoss', binary_ins=False, loss_weight=0.25, loss_type='binary_cross_entropy')),
                   dict(loss_mil='AllPosLoss', mil_loss_type='binary_cross_entropy'), False),
    'mil_bce_variants': (dict(loss_mil=dict(type='MILLoss', binary_ins=True, loss_weight=0.25, loss_type='binary_cross_entropy'),
                              normal_cfg=dict(prob_cls_type='softmax', out_bg_cls=False)),
                         dict(mil_loss_type='binary_cross_entropy', binary_ins=True, prob_cls_type='softmax'), True),
}


def loss_type_inputs(case, seed=SEED):
    """CPR-lite inputs + one GT centred outside pad_shape by more than the ring radius (every bag sample invalid); the variant case gets
    a doubled instance classifier (binary_ins) and gt_weights with a zero weight on the first GT.  returns (inp, weights, gt_weights)."""
    inp = synth.cpr_inputs('lite', seed, trained_like=True)
    d = inp['cfgd']
    ph, pw = d['pad_hw']
    reach = d['radius'] * d['stride']
    out_pt = torch.tensor([[pw + reach + 24.0, 0.5 * ph]])
    inp['gt_bboxes'][0] = torch.cat([inp['gt_bboxes'][0], torch.cat([out_pt - 8, out_pt + 8], dim=1)])
    inp['gt_labels'][0] = torch.cat([inp['gt_labels'][0], torch.tensor([3])])
    inp['gt_anns_id'][0] = torch.arange(len(inp['gt_labels'][0]))
    w = dict(inp['weights'])
    gtw = None
    if LOSS_TYPE_CASES[case][2]:
        g = torch.Generator().manual_seed(seed + 23)
        n, C = d['num_classes'], d['C']
        w['ins_out.weight'] = torch.cat([w['ins_out.weight'], torch.randn(n, C, generator=g) * 0.05])
        w['ins_out.bias'] = torch.cat([w['ins_out.bias'], torch.zeros(n)])
        gtw = [torch.rand(len(l), generator=g) * 0.5 + 0.5 for l in inp['gt_labels']]
        gtw[0][0] = 0.0                                                          # a bag whose weight is zero
    return inp, w, gtw


def oracle_cfg(case, d):
    return ocpr.default_cfg(num_classes=d['num_classes'], in_channels=d['C'], feat_channels=d['C'], stride=d['stride'],
                            pos_radius=d['radius'], neg_radius=d['radius'], **LOSS_TYPE_CASES[case][1])


def label_margin(prob, labels):
    """min over rows of |p[label] - max_{c != label} p[c]|: how far each top-1 hit is from flipping.  Rows whose probabilities are
    all equal (the fully invalid bag: prob = 0 exactly) are a tie by construction; they must be misses both for the reference's topk
    and for the first-maximum rule (class 0), so their label must not be 0 or what topk returns."""
    p = prob.detach().double().clone()
    const = p.max(dim=1)[0] == p.min(dim=1)[0]
    assert not (labels[const] == 0).any() and not (prob[const].topk(1, dim=1)[1][:, 0] == labels[const]).any(), 'constant row scored a hit'
    pl = p[torch.arange(len(p)), labels].clone()
    p[torch.arange(len(p)), labels] = -1.0
    return float((pl - p.max(dim=1)[0])[~const].abs().min())


def golden_loss_type(HEADS, case, seed=SEED):
    inp, w, gtw = loss_type_inputs(case, seed)
    d = inp['cfgd']
    rcfg = ref_cpr_cfg(d)
    rcfg.update(LOSS_TYPE_CASES[case][0])
    head = HEADS.build(rcfg)
    sd = head.state_dict()
    for k in sd:
        if k.startswith('cls_convs'):
            w[k] = sd[k]
    head.load_state_dict(w, strict=True)
    head.eval()
    cfg = oracle_cfg(case, d)
    gtb, gtl, metas = inp['gt_bboxes'], inp['gt_labels'], inp['img_metas']
    # ---- reference: losses reduced like mmdet's _parse_losses (AllPosLoss returns loss + bag_ins_outs * 0, a tensor)
    f_ref = inp['cls_feat'].clone().requires_grad_(True)
    rl = head.loss([f_ref], [f_ref], gtb, gtl, metas, gt_weights=gtw)
    rl = {k: v.mean() if 'loss' in k else v for k, v in rl.items()}
    sum(v for k, v in rl.items() if 'loss' in k).backward()
    # ---- oracle
    f_o = inp['cls_feat'].clone().requires_grad_(True)
    wo = {k: v.clone().requires_grad_(True) for k, v in w.items() if not k.startswith('cls_convs')}
    ol, oall = olt.cpr_loss(f_o, wo, gtb, gtl, metas, cfg, return_all=True, gt_weights=gtw)
    sum(v for k, v in ol.items() if 'loss' in k).backward()
    out = {}
    for k in ('gt_loss', 'pos_loss', 'neg_loss', 'bag_acc'):
        eq(ol[k].detach().reshape(-1), rl[k].detach().reshape(-1), f'{case} {k}', exact=False, tol=1e-6)
        out['loss_' + k] = rl[k].detach().reshape(-1).numpy()
    eq(f_o.grad, f_ref.grad, f'{case} dfeat', exact=False, tol=1e-6)
    for name in ('cls_out.weight', 'cls_out.bias', 'ins_out.weight', 'ins_out.bias'):
        mod, p = name.split('.')
        eq(wo[name].grad, getattr(getattr(head, mod), p).grad, f'{case} d{name}', exact=False, tol=1e-6)
        out['grad_' + mod.split('_')[0] + '_' + p[0]] = getattr(getattr(head, mod), p).grad.numpy()
    if cfg.get('loss_mil', 'MILLoss') == 'AllPosLoss':
        assert not head.ins_out.weight.grad.any() and not head.ins_out.bias.grad.any(), 'AllPosLoss: instance gradient not zero'
    # ---- near-tie guard for bag_acc
    labels = torch.cat(gtl)
    with torch.no_grad():
        if cfg.get('loss_mil', 'MILLoss') == 'AllPosLoss':
            K = oall['pos_cls'].shape[2]
            prob = ocpr.cls_prob(oall['pos_cls'], cfg).reshape(len(labels) * K, -1)
            m = label_margin(prob, labels.repeat_interleave(K))
        else:
            m = label_margin(oall['bag_prob'], labels)
    assert m > TIE, f'{case}: a top-1 decision within {m:.2e} of a tie; pick another seed'
    out['grad_feat_sub'], out['grad_feat_sum'], out['grad_feat_abs'] = sub(f_ref.grad, 211)
    out['label_margin'] = np.float64(m)
    out['seed'] = np.int64(seed)
    path = os.path.join(GOLD, f'cpr_lite_loss_{case}.npz')
    np.savez_compressed(path, **out)
    print(f'[golden] {path}: ' + ' '.join(f'{k}={float(v.detach().reshape(-1)[0]):.6f}' for k, v in rl.items() if v is not None) + f'; label margin {m:.2e}')


def main():
    torch.set_num_threads(max(1, min(8, os.cpu_count() or 1)))
    HEADS = load_reference()
    for case in LOSS_TYPE_CASES:
        golden_loss_type(HEADS, case)


if __name__ == '__main__':
    main()
