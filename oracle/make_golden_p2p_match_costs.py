"""Pins oracle/p2p_match_costs.py against the REAL reference and writes tests/golden/p2p_match_costs.npz.  (test infrastructure)

Run in the build container only (needs /root/reference):   python -m oracle.make_golden_p2p_match_costs
The unmodified reference mmdet package is imported through oracle/_mmcv_stub.py.  For each cost set the real HungarianAssignerV2 is
built from its config, its own cost lists are summed as assign() sums them (hungarian_assigner.py:223-227) and the oracle's cost is
ASSERTED bit-identical; assign() then runs at topk_k 1 and 5 and its assignments are stored.  A head-level case runs the real
P2PHead.loss (softmax CrossEntropyLoss) with the paper's costs, ClassificationCostV2(use_sigmoid=False) + DisCostV2(p=2).

Tie guard: every stored assignment is asserted unchanged when scipy runs on the reference cost times (1 + 1e-6 u), u uniform in
[-1, 1], over several seeded draws, so that the CUDA cost's few-ulp softmax and sqrt differences cannot flip a match.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import p2p as op2p, p2p_softmax as osm, p2p_match_costs as omc  # noqa: E402
from oracle._mmcv_stub import load_reference, CfgDict  # noqa: E402
from oracle.make_golden import GOLD, eq, sub  # noqa: E402
from oracle.p2p_match_costs import CASES, IMG_SHAPE, PAPER  # noqa: E402

SEED = 9031
TIE_REL, TIE_DRAWS = 1e-6, 8
HEAD_TRAIN_CFG = dict(neg_weight=1.0, assigner=dict(type='HungarianAssignerV2', cls_costs=omc.cost_config(PAPER)[0],
                                                    reg_costs=omc.cost_config(PAPER)[1], topk_k=5),
                      sampler=dict(type='PseudoSampler'))


def case_inputs(seed, N, n, C1):
    g = torch.Generator().manual_seed(seed)
    h, w = IMG_SHAPE[:2]
    pts = torch.rand(N, 2, generator=g) * torch.tensor([w, h])
    cls = torch.randn(N, C1, generator=g) * 2.0
    gts = torch.rand(n, 2, generator=g) * torch.tensor([w, h])
    labels = torch.randint(0, min(C1, 80), (n,), generator=g)
    return pts, cls, gts, labels


def tie_guard(cost, gt_inds, gt_labels, topk_k, what, seed):
    g = torch.Generator().manual_seed(seed)
    for d in range(TIE_DRAWS):
        u = torch.rand(cost.shape, generator=g, dtype=torch.float64) * 2 - 1
        gi, _ = op2p.hungarian_v2_from_cost(cost.double() * (1 + TIE_REL * u), gt_labels, topk_k)
        assert torch.equal(gi, gt_inds), f'{what}: assignment flips under a 1e-6 relative perturbation (draw {d})'


def golden_cost_sets(out):
    from mmdet.core.bbox.assigners.hungarian_assigner import HungarianAssignerV2
    for ci, (name, (terms, N, n, C1)) in enumerate(CASES.items()):
        pts, cls, gts, labels = case_inputs(SEED + ci, N, n, C1)
        meta = dict(img_shape=IMG_SHAPE)
        cc, rc = omc.cost_config(terms)
        ref = HungarianAssignerV2(cls_costs=cc, reg_costs=rc, topk_k=1)
        cost_r = sum([c(cls, labels) for c in ref.cls_costs]) + sum([c(pts, gts, meta) for c in ref.reg_costs])
        cost_o = omc.cost_matrix(pts, cls, gts, labels, IMG_SHAPE, terms)
        eq(cost_o, cost_r, f'{name} cost')
        out[f'{name}_pts'], out[f'{name}_cls'], out[f'{name}_gts'] = pts.numpy(), cls.numpy(), gts.numpy()
        out[f'{name}_labels'], out[f'{name}_cost'] = labels.numpy(), cost_r.numpy()
        for k in (1, 5):
            ref.topk_k = k
            res = ref.assign(pts, cls, gts, labels, meta)
            gi, _ = op2p.hungarian_v2_from_cost(cost_o, labels, k)
            eq(gi, res.gt_inds, f'{name} topk {k} gt_inds')
            tie_guard(cost_r, res.gt_inds, labels, k, f'{name} topk {k}', SEED + 100 * ci + k)
            out[f'{name}_gt_inds_k{k}'] = res.gt_inds.numpy().astype(np.int32)
        print(f'[golden] {name}: {N} x {n}, {C1} columns, {int((out[f"{name}_gt_inds_k5"] > 0).sum())} matches at topk_k 5')


def golden_head(HEADS, out, seed=4267):
    """the real P2PHead.loss with softmax CrossEntropyLoss and the paper costs, on the oracle's head outputs of the softmax case"""
    import mmdet.models.point.dense_heads.p2p_head as ref_mod
    ref_mod.TestP2PHead.test_assign = staticmethod(lambda *a, **k: None)   # debug visualiser (needs huicv)
    inp = osm.inputs(seed)
    d = inp['cfgd']
    C = d['num_classes']
    metas, gtb, gtl = inp['img_metas'], inp['gt_bboxes'], inp['gt_labels']
    head = HEADS.build(dict(type='P2PHead', num_classes=C, in_channels=d['C'], feat_channels=d['C'], stacked_convs=4,
                            strides=[d['stride']], norm_cfg=dict(type='GN', num_groups=32, requires_grad=True),
                            loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0),
                            train_cfg=CfgDict(HEAD_TRAIN_CFG), test_cfg=CfgDict(dict(nms_pre=200))))
    cfg = osm.softmax_cfg(use_sigmoid=False, num_classes=C, stride=d['stride'])
    with torch.no_grad():
        oc, opo = op2p.head_forward(inp['x'], inp['weights'], cfg)
        _, rpd, rv, rcl = head.get_pred_points([oc], [opo], metas)
        gt_points = head.pseudo_bbox_to_center(gtb)
        rl = head.get_targets(rpd[..., :2], rv, rcl, gt_points, gtl, metas, None)[0]
        _, opd, ov, ocl = osm.pred_points(oc, opo, metas, cfg)
    gis, lbs = [], []
    for b in range(len(metas)):
        v = ov[b]
        props, cl = opd[b][..., :2][v], ocl[b][v]
        cost = omc.cost_matrix(props, cl, gt_points[b], gtl[b], metas[b]['img_shape'], PAPER)
        gi_v, _ = op2p.hungarian_v2_from_cost(cost, gtl[b], 5)
        tie_guard(cost, gi_v, gtl[b], 5, f'head image {b}', seed + b)
        gi = torch.zeros(v.shape[0], dtype=torch.long)
        gi[v] = gi_v
        lab = torch.where(gi > 0, gtl[b][(gi - 1).clamp(min=0)], torch.full_like(gi, C))
        lab = torch.where(v, lab, torch.zeros_like(lab))
        eq(lab, rl[b], f'head labels image {b}')
        gis.append(gi); lbs.append(lab)
    out['head_gt_inds'] = torch.stack(gis).numpy().astype(np.int32)
    out['head_labels'] = torch.stack(lbs).numpy()
    co, po = oc.clone().requires_grad_(True), opo.clone().requires_grad_(True)
    rloss = head.loss([co], [po], gtb, gtl, metas, gt_bboxes_ignore=[torch.zeros(0, 4) for _ in metas])
    (sum(rloss['loss_cls']) + sum(rloss['loss_pts'])).backward()
    for k in ('loss_cls', 'loss_pts'):
        out['head_' + k] = torch.stack(rloss[k]).detach().numpy()
    out['head_grad_cls_sub'], out['head_grad_cls_sum'], _ = sub(co.grad, 37)
    out['head_grad_pts_sub'], out['head_grad_pts_sum'], _ = sub(po.grad, 1)
    out['head_seed'] = np.int64(seed)
    print(f'[golden] head: pos {int((out["head_gt_inds"] > 0).sum())}; loss_cls {out["head_loss_cls"].tolist()} '
          f'loss_pts {out["head_loss_pts"].tolist()}')


def main():
    torch.set_num_threads(os.cpu_count())
    os.makedirs(GOLD, exist_ok=True)
    HEADS = load_reference()
    out = {}
    golden_cost_sets(out)
    golden_head(HEADS, out)
    out['seed'] = np.int64(SEED)
    path = os.path.join(GOLD, 'p2p_match_costs.npz')
    np.savez_compressed(path, **out)
    print(f'[golden] {path}: {os.path.getsize(path) / 1024:.0f} KiB')


if __name__ == '__main__':
    main()
