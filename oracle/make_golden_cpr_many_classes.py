"""Pins the oracle against the REAL reference CPRHead at 365 and 1203 classes (Objects365's and LVIS's class counts) and writes
tests/golden/cpr_many_classes_<N>.npz.  (test infrastructure)

Run in the build container only (needs /root/reference):   python -m oracle.make_golden_cpr_many_classes
Same procedure as oracle/make_golden.py::golden_cpr_variant: the unmodified reference CPRHead is built through oracle/_mmcv_stub.py from
oracle/make_golden.py's config with num_classes = N, reference and oracle run the loss, its backward and get_bboxes on the same seeded
inputs, their equality is ASSERTED (1e-6), then the reference's outputs are stored.  The inputs are CPR-lite (one 256 x 256 image, stride 8)
at 32 feature channels with 12 GTs, plus one GT at (2, 3) whose ring bag lies partly outside pad_shape, so the fixtures stay small.
The inputs are asserted free of bag_acc near-ties (oracle/make_golden_cpr_loss_types.py::label_margin).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import cpr as ocpr, synth  # noqa: E402
from oracle._mmcv_stub import load_reference  # noqa: E402
from oracle.make_golden import GOLD, eq, ref_cpr_cfg, sub  # noqa: E402
from oracle.make_golden_cpr_loss_types import TIE, label_margin  # noqa: E402

CLASS_COUNTS = (365, 1203)
SEEDS = {365: 3650, 1203: 12030}
C_FEAT = 32
N_GT = 12


def many_class_inputs(N, seed=None):
    """CPR-lite inputs at N classes and 32 channels, 12 GTs and one more GT centred at (2, 3): part of its ring bag is outside pad_shape."""
    seed = SEEDS[N] if seed is None else seed
    inp = synth.cpr_inputs('lite', seed, trained_like=True, num_classes=N, C=C_FEAT, n=N_GT)
    edge = torch.tensor([[2.0, 3.0]])
    inp['gt_bboxes'][0] = torch.cat([inp['gt_bboxes'][0], torch.cat([edge - 8, edge + 8], dim=1)])
    inp['gt_labels'][0] = torch.cat([inp['gt_labels'][0], torch.tensor([N - 1])])
    inp['gt_anns_id'][0] = torch.arange(len(inp['gt_labels'][0]))
    return inp


def oracle_cfg(d):
    return ocpr.default_cfg(num_classes=d['num_classes'], in_channels=d['C'], feat_channels=d['C'], stride=d['stride'],
                            pos_radius=d['radius'], neg_radius=d['radius'])


def golden_many_classes(HEADS, N):
    inp = many_class_inputs(N)
    d = inp['cfgd']
    head = HEADS.build(ref_cpr_cfg(d))
    w = dict(inp['weights'])
    sd = head.state_dict()
    for k in sd:
        if k.startswith('cls_convs'):
            w[k] = sd[k]
    head.load_state_dict(w, strict=True)
    head.eval()
    cfg = oracle_cfg(d)
    gtb, gtl, metas, aid = inp['gt_bboxes'], inp['gt_labels'], inp['img_metas'], inp['gt_anns_id']
    f_ref = inp['cls_feat'].clone().requires_grad_(True)
    rl = head.loss([f_ref], [f_ref], gtb, gtl, metas)
    sum(v for k, v in rl.items() if 'loss' in k).backward()
    f_o = inp['cls_feat'].clone().requires_grad_(True)
    wo = {k: v.clone().requires_grad_(True) for k, v in w.items() if not k.startswith('cls_convs')}
    ol, oall = ocpr.cpr_loss(f_o, wo, gtb, gtl, metas, cfg, return_all=True)
    sum(v for k, v in ol.items() if 'loss' in k).backward()
    out = {}
    for k in ('gt_loss', 'pos_loss', 'neg_loss', 'bag_acc'):
        eq(ol[k].detach().reshape(-1), rl[k].detach().reshape(-1), f'N={N} {k}', exact=False, tol=1e-6)
        out['loss_' + k] = rl[k].detach().reshape(-1).numpy()
    eq(f_o.grad, f_ref.grad, f'N={N} dfeat', exact=False, tol=1e-6)
    for name in ('cls_out.weight', 'cls_out.bias', 'ins_out.weight', 'ins_out.bias'):
        mod, p = name.split('.')
        eq(wo[name].grad, getattr(getattr(head, mod), p).grad, f'N={N} d{name}', exact=False, tol=1e-6)
        out['grad_' + mod.split('_')[0] + '_' + p[0]] = getattr(getattr(head, mod), p).grad.numpy()
    out['grad_feat_sub'], out['grad_feat_sum'], out['grad_feat_abs'] = sub(f_ref.grad, 211)
    out['mil_bag_prob'] = oall['bag_prob'].detach().numpy()
    m = label_margin(oall['bag_prob'], torch.cat(gtl))
    assert m > TIE, f'N={N}: a top-1 decision within {m:.2e} of a tie; pick another seed'
    out['label_margin'] = np.float64(m)
    out['pos_valid'] = oall['ex']['pos_valid'].numpy()
    assert not bool(out['pos_valid'][-1].all()) and bool(out['pos_valid'][-1].any()), 'the edge GT must have a partly valid bag'
    with torch.no_grad():
        rres = head.get_bboxes([inp['cls_feat']], [inp['cls_feat']], metas, gt_bboxes=gtb, gt_labels=gtl, gt_anns_id=aid)
        ores, orall = ocpr.cpr_get_bboxes(inp['cls_feat'], w, gtb, gtl, aid, metas, cfg, return_all=True)
    for b in range(len(rres)):
        eq(ores[b][0], rres[b][0], f'N={N} det[{b}]')
    out['det'] = torch.cat([r[0] for r in rres]).numpy()
    out['not_refine'] = torch.cat([r['not_refine'] for r in orall['refine']]).numpy()
    out['chosen'] = torch.cat([r['chosen'] for r in orall['refine']]).numpy()
    out['seed'] = np.int64(SEEDS[N])
    path = os.path.join(GOLD, f'cpr_many_classes_{N}.npz')
    np.savez_compressed(path, **out)
    print(f'[golden] {path}: {os.path.getsize(path) / 1024:.0f} KiB; losses '
          + ' '.join(f'{k}={float(v.reshape(-1)[0]):.6f}' for k, v in rl.items()) + f'; not_refine {float(out["not_refine"].mean()):.2f}')


def main():
    torch.set_num_threads(max(1, min(8, os.cpu_count() or 1)))
    HEADS = load_reference()
    for N in CLASS_COUNTS:
        golden_many_classes(HEADS, N)


if __name__ == '__main__':
    main()
