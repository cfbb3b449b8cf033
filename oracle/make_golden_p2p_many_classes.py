"""Pins the P2P oracles against the REAL reference P2PHead at 365 and 1203 classes (Objects365's and LVIS's class counts), where cls_out
is wider than one 512-channel conv launch, and writes tests/golden/p2p_many_classes_<case>.npz.  (test infrastructure)

Run in the build container only (needs /root/reference):   python -m oracle.make_golden_p2p_many_classes
Same procedure and helpers as oracle/make_golden_p2p_defaults.py and make_golden_p2p_softmax.py: the unmodified reference mmdet package
is imported through oracle/_mmcv_stub.py, each head is built, reference and oracle (oracle/p2p.py, p2p_defaults.py, p2p_softmax.py, used
as is: they take any channel count) run the whole head (towers, output convs, loss, backward into the input and the weights, get_bboxes)
on the same seeded inputs, their equality is ASSERTED (1e-6), then the reference's outputs are stored.  The cases:
  defaults_365 / defaults_1203  the reference class's own defaults (4 anchors, CrossEntropyLoss(use_sigmoid=True) + MSELoss):
                                cls_out 1460 / 4812 channels
  shipped_1203                  the shipped configs' head (one anchor, FocalLoss + SmoothL1Loss): 1203 channels, not a multiple of 4
  softmax_365                   softmax CrossEntropyLoss with class_weight: 4 x 366 = 1464 channels, background last per anchor
Inputs are oracle/p2p_defaults.py's (p2p_softmax.py's for the softmax case) at 10 GT points per image on a 16 x 16 map; the shipped head
takes anchor 0's rows of the default weights.  To keep each fixture under 400 KB the maps and the input gradient are stored as strided
samples with float64 checksums, and the cls_out weight gradient as a seeded subset of rows (the first, the last and, in softmax mode,
every background row).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import p2p as op2p, p2p_defaults as odef, p2p_softmax as osm  # noqa: E402
from oracle._mmcv_stub import load_reference, CfgDict  # noqa: E402
from oracle.make_golden import GOLD, eq, sub  # noqa: E402
from oracle.make_golden_p2p_defaults import P2P_DEFAULTS_TRAIN_CFG, P2P_DEFAULTS_TEST_CFG  # noqa: E402
from oracle.make_golden_p2p_softmax import class_weights  # noqa: E402

CASES = {
    'defaults_365': dict(kind='defaults', num_classes=365, seed=3651),
    'defaults_1203': dict(kind='defaults', num_classes=1203, seed=12031),
    'shipped_1203': dict(kind='shipped', num_classes=1203, seed=12032),
    'softmax_365': dict(kind='softmax', num_classes=365, seed=3652),
}
N_POINTS = 10
MAP_STEP, GRAD_X_STEP, N_SEEDED_ROWS = 211, 37, 6
SHIPPED_LOSSES = dict(loss_cls=dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0),
                      loss_reg=dict(type='SmoothL1Loss', beta=1.0 / 9.0, loss_weight=0.5))


def case_inputs(name):
    """(inputs, oracle cfg, reference / product head kwargs) of one case."""
    c = CASES[name]
    N, kind = c['num_classes'], c['kind']
    if kind == 'softmax':
        inp = osm.inputs(c['seed'], num_classes=N, n=N_POINTS)
        cw, _ = class_weights(N)
        cfg = osm.softmax_cfg(use_sigmoid=False, class_weight=cw, num_classes=N, stride=inp['cfgd']['stride'], nms_iou=0.5)
        head_kw = dict(loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=False, class_weight=cw, loss_weight=1.0))
        return inp, cfg, head_kw
    inp = odef.inputs(c['seed'], num_classes=N, n=N_POINTS)
    stride = inp['cfgd']['stride']
    if kind == 'defaults':
        return inp, odef.reference_defaults_cfg(num_classes=N, stride=stride, nms_iou=0.5), {}
    w = inp['weights']                          # shipped: one anchor at the cell corner, anchor 0's rows of the default weights
    for k, n in (('cls_out', N), ('reg_out', 2)):
        w[f'{k}.weight'], w[f'{k}.bias'] = w[f'{k}.weight'][:n].contiguous(), w[f'{k}.bias'][:n].contiguous()
    inp['cfgd']['point_anchor'] = [(0., 0.)]
    cfg = odef.reference_defaults_cfg(num_classes=N, stride=stride, nms_iou=0.5, point_anchor=[(0., 0.)], pts_gamma=1.0, reg_norm=1.0,
                                      loss_cls='FocalLoss', loss_reg='SmoothL1Loss', loss_reg_weight=0.5)
    return inp, cfg, dict(point_anchor=[(0., 0.)], pts_gamma=1, reg_norm=1, **SHIPPED_LOSSES)


def weight_rows(name, n_out, k):
    """rows of the cls_out weight gradient a fixture keeps: the first, the last, the background row of every anchor in softmax mode,
    and N_SEEDED_ROWS more drawn from the case's seed."""
    rows = {0, n_out - 1}
    if CASES[name]['kind'] == 'softmax':
        c1 = n_out // k
        rows |= {a * c1 + c1 - 1 for a in range(k)}
    gen = torch.Generator().manual_seed(CASES[name]['seed'])
    rows |= set(torch.randint(0, n_out, (N_SEEDED_ROWS,), generator=gen).tolist())
    return np.array(sorted(rows), dtype=np.int64)


def oracle_loss(name):
    return osm.p2p_loss if CASES[name]['kind'] == 'softmax' else odef.p2p_loss


def oracle_bboxes_single(name):
    return osm.get_bboxes_single if CASES[name]['kind'] == 'softmax' else op2p.get_bboxes_single


def oracle_pred_points(name):
    return osm.pred_points if CASES[name]['kind'] == 'softmax' else op2p.pred_points


def golden_case(HEADS, name):
    import mmdet.models.point.dense_heads.p2p_head as ref_mod
    ref_mod.TestP2PHead.test_assign = staticmethod(lambda *a, **k: None)   # debug visualiser (needs huicv)
    inp, cfg, head_kw = case_inputs(name)
    d = inp['cfgd']
    k = len(cfg['point_anchor'])
    head = HEADS.build(dict(type='P2PHead', num_classes=d['num_classes'], in_channels=d['C'], feat_channels=d['C'], stacked_convs=4,
                            strides=[d['stride']], norm_cfg=dict(type='GN', num_groups=32, requires_grad=True),
                            train_cfg=CfgDict(P2P_DEFAULTS_TRAIN_CFG), test_cfg=CfgDict(P2P_DEFAULTS_TEST_CFG), **head_kw))
    n_out = head.cls_out.out_channels
    assert head.num_points == k and n_out > 512, (head.num_points, n_out)
    head.load_state_dict(inp['weights'], strict=True)
    head.eval()
    gtb, gtl, metas = inp['gt_bboxes'], inp['gt_labels'], inp['img_metas']
    ign = [torch.zeros(0, 4) for _ in metas]
    out = {}
    # ---- forward + loss + backward into the input and every weight, reference and oracle
    x_r = inp['x'].clone().requires_grad_(True)
    rc, rp = head((x_r,))
    rc, rp = rc[0], rp[0]
    rloss = head.loss([rc], [rp], gtb, gtl, metas, gt_bboxes_ignore=ign)
    (sum(rloss['loss_cls']) + sum(rloss['loss_pts'])).backward()
    x_o = inp['x'].clone().requires_grad_(True)
    wo = {kk: v.clone().requires_grad_(True) for kk, v in inp['weights'].items()}
    oc, opo = op2p.head_forward(x_o, wo, cfg)
    eq(oc, rc, 'cls_out', exact=False, tol=1e-6)
    eq(opo, rp, 'pts_out', exact=False, tol=1e-6)
    oloss, oall = oracle_loss(name)(oc, opo, gtb, gtl, metas, cfg, return_all=True)
    (sum(oloss['loss_cls']) + sum(oloss['loss_pts'])).backward()
    for kk in ('loss_cls', 'loss_pts'):
        eq(torch.stack(oloss[kk]).detach(), torch.stack(rloss[kk]).detach(), kk, exact=False, tol=1e-6)
        out[kk] = torch.stack(rloss[kk]).detach().numpy()
    eq(x_o.grad, x_r.grad, 'dx', exact=False, tol=1e-6)
    for p in ('cls_out.weight', 'cls_out.bias', 'reg_out.weight', 'reg_out.bias'):
        mod, attr = p.split('.')
        eq(wo[p].grad, getattr(getattr(head, mod), attr).grad, f'd{p}', exact=False, tol=1e-6)
    out['gt_inds'] = torch.stack([t[4] for t in oall['targets']]).numpy().astype(np.int32)
    rc, rp = rc.detach(), rp.detach()
    out['cls_out_sub'], out['cls_out_sum'], out['cls_out_abs'] = sub(rc, MAP_STEP)
    out['pts_out_sub'], out['pts_out_sum'], out['pts_out_abs'] = sub(rp, 1)
    out['grad_x_sub'], out['grad_x_sum'], out['grad_x_abs'] = sub(x_r.grad, GRAD_X_STEP)
    rows = weight_rows(name, n_out, k)
    out['grad_w_cls_rows'] = rows
    out['grad_w_cls'] = head.cls_out.weight.grad[torch.from_numpy(rows)].numpy()
    out['grad_b_cls'] = head.cls_out.bias.grad.numpy()
    out['grad_w_reg'] = head.reg_out.weight.grad.numpy()
    out['grad_b_reg'] = head.reg_out.bias.grad.numpy()
    # ---- get_bboxes of the reference against the oracle's decode + top-k + multiclass_nms
    with torch.no_grad():
        rres = head.get_bboxes([rc], [rp], metas)
        _, opd, _, ocl = oracle_pred_points(name)(rc, rp, metas, cfg)
        dets, labs, keeps, cands, topks = [], [], [], [], []
        for b in range(len(metas)):
            ps, labels, al = oracle_bboxes_single(name)(opd[b][..., :2], ocl[b], metas[b]['img_shape'], metas[b]['scale_factor'], cfg,
                                                        return_all=True)
            wh = torch.tensor(cfg['pseudo_wh'])
            eq(torch.cat([ps[:, :2] - wh / 2, ps[:, :2] + wh / 2, ps[:, 2:]], -1), rres[b][0], f'{name} det[{b}]')
            eq(labels, rres[b][1], f'{name} labels[{b}]')
            dets.append(rres[b][0]); labs.append(rres[b][1]); keeps.append(al['keep']); cands.append(al['cand_inds'])
            topks.append(al['topk_inds'] if al['topk_inds'] is not None else torch.zeros(0, dtype=torch.long))
    out['det_len'] = np.array([len(x) for x in dets])
    out['det'] = torch.cat(dets).numpy()
    out['det_labels'] = torch.cat(labs).numpy()
    out['keep'] = torch.cat(keeps).numpy()
    out['cand_len'] = np.array([len(x) for x in cands])
    out['topk'] = torch.cat(topks).numpy().astype(np.int32)
    out['seed'] = np.int64(CASES[name]['seed'])
    path = os.path.join(GOLD, f'p2p_many_classes_{name}.npz')
    np.savez_compressed(path, **out)
    print(f'[golden] {path}: {os.path.getsize(path) / 1024:.0f} KiB; cls_out {n_out} channels; dets/img {out["det_len"].tolist()} '
          f'cands/img {out["cand_len"].tolist()} pos {int((out["gt_inds"] > 0).sum())}; losses cls {out["loss_cls"].tolist()} '
          f'pts {out["loss_pts"].tolist()}')
    assert os.path.getsize(path) < 400 * 1024, path


def main():
    torch.set_num_threads(max(1, min(8, os.cpu_count() or 1)))
    os.makedirs(GOLD, exist_ok=True)
    HEADS = load_reference()
    for name in CASES:
        golden_case(HEADS, name)


if __name__ == '__main__':
    main()
