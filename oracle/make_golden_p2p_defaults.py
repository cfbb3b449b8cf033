"""Pins oracle/p2p_defaults.py against the REAL reference and writes tests/golden/p2p_defaults_lite.npz.  (test infrastructure)

Run in the build container only (needs /root/reference):   python -m oracle.make_golden_p2p_defaults
Same procedure and helpers as oracle/make_golden.py (which writes every other fixture): the unmodified reference mmdet package is
imported through oracle/_mmcv_stub.py, P2PHead is built from its OWN defaults, reference and oracle run on the same seeded inputs and
their equality is ASSERTED before the reference's outputs are stored.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import p2p as op2p, p2p_defaults as odef  # noqa: E402
from oracle._mmcv_stub import load_reference, CfgDict  # noqa: E402
from oracle.make_golden import GOLD, eq, sub  # noqa: E402


P2P_DEFAULTS_TRAIN_CFG = dict(neg_weight=1.0, assigner=dict(type='HungarianAssignerV2', cls_costs=dict(type='FocalLossCost', weight=2.0),
                                                             reg_costs=dict(type='DisCostV2', weight=0.1, norm_with_img_wh=False),
                                                             topk_k=5), sampler=dict(type='PseudoSampler'))
P2P_DEFAULTS_TEST_CFG = dict(nms_pre=1000, min_bbox_size=0, score_thr=0.05, pseudo_wh=(32, 32), nms=dict(type='nms', iou_threshold=0.5),
                             max_per_img=100)


def golden_p2p_defaults(HEADS, seed=8086):
    """P2PHead at the reference class's OWN defaults (p2p_head.py:25-45: four point anchors per cell, pts_gamma 100/8, reg_norm 1/8,
    CrossEntropyLoss(use_sigmoid=True) + MSELoss(loss_weight=2e-4)): no anchor or loss kwargs, only the GroupNorm towers, one stride
    and the train / test settings every config sets.  80 classes x 4 anchors = 320 cls_out channels.  Towers + output convs, loss
    (+ gradients w.r.t. the two output maps) and get_bboxes of the REAL head vs the oracle on seeded weights / inputs."""
    import mmdet.models.point.dense_heads.p2p_head as ref_mod
    ref_mod.TestP2PHead.test_assign = staticmethod(lambda *a, **k: None)   # debug visualiser (needs huicv)
    inp = odef.inputs(seed)
    d = inp['cfgd']
    head = HEADS.build(dict(type='P2PHead', num_classes=d['num_classes'], in_channels=d['C'], feat_channels=d['C'], stacked_convs=4,
                            strides=[d['stride']], norm_cfg=dict(type='GN', num_groups=32, requires_grad=True),
                            train_cfg=CfgDict(P2P_DEFAULTS_TRAIN_CFG), test_cfg=CfgDict(P2P_DEFAULTS_TEST_CFG)))
    assert head.num_points == 4 and head.cls_out.out_channels == 4 * d['num_classes'], (head.num_points, head.cls_out)
    assert type(head.loss_cls).__name__ == 'CrossEntropyLoss' and type(head.loss_reg).__name__ == 'MSELoss'
    head.load_state_dict(inp['weights'], strict=True)
    head.eval()
    cfg = odef.reference_defaults_cfg(num_classes=d['num_classes'], stride=d['stride'], nms_iou=0.5)
    assert [tuple(a) for a in head.point_anchor.tolist()] == [tuple(a) for a in cfg['point_anchor']]
    assert (head.pts_gamma, head.reg_norm, head.loss_reg.loss_weight) == (cfg['pts_gamma'], cfg['reg_norm'], cfg['loss_reg_weight'])
    gtb, gtl, metas = inp['gt_bboxes'], inp['gt_labels'], inp['img_metas']
    out = {}
    with torch.no_grad():
        rc, rp = head((inp['x'],))
        rc, rp = rc[0], rp[0]
        oc, opo = op2p.head_forward(inp['x'], inp['weights'], cfg)
    eq(oc, rc, 'cls_out', exact=False, tol=1e-6)
    eq(opo, rp, 'pts_out', exact=False, tol=1e-6)
    out['cls_out_sub'], out['cls_out_sum'], out['cls_out_abs'] = sub(rc, 37)
    out['pts_out_sub'], out['pts_out_sum'], out['pts_out_abs'] = sub(rp, 1)
    with torch.no_grad():
        _, rpd, rv, rcl = head.get_pred_points([rc], [rp], metas)
        gt_points = head.pseudo_bbox_to_center(gtb)
        rl, rlw, rgp, rpw = head.get_targets(rpd[..., :2], rv, rcl, gt_points, gtl, metas, None)
        _, opd, ov, ocl = op2p.pred_points(rc, rp, metas, cfg)
        tg = [op2p.target_single(opd[b][..., :2], ov[b], ocl[b], gt_points[b], gtl[b], metas[b]['img_shape'], cfg)
              for b in range(len(metas))]
        for b in range(len(metas)):
            eq(tg[b][0], rl[b], 'labels'); eq(tg[b][1], rlw[b], 'lw'); eq(tg[b][2], rgp[b], 'gpts'); eq(tg[b][3], rpw[b], 'pw')
        out['gt_inds'] = torch.stack([t[4] for t in tg]).numpy().astype(np.int32)
    co_r, po_r = rc.clone().requires_grad_(True), rp.clone().requires_grad_(True)
    rloss = head.loss([co_r], [po_r], gtb, gtl, metas, gt_bboxes_ignore=[torch.zeros(0, 4) for _ in metas])
    (sum(rloss['loss_cls']) + sum(rloss['loss_pts'])).backward()
    co, po = rc.clone().requires_grad_(True), rp.clone().requires_grad_(True)
    oloss = odef.p2p_loss(co, po, gtb, gtl, metas, cfg)
    (sum(oloss['loss_cls']) + sum(oloss['loss_pts'])).backward()
    for k in ('loss_cls', 'loss_pts'):
        eq(torch.stack(oloss[k]).detach(), torch.stack(rloss[k]).detach(), k, exact=False, tol=1e-6)
        out[k] = torch.stack(rloss[k]).detach().numpy()
    eq(co.grad, co_r.grad, 'dcls', exact=False, tol=1e-6)
    eq(po.grad, po_r.grad, 'dpts', exact=False, tol=1e-6)
    out['grad_cls_sub'], out['grad_cls_sum'], out['grad_cls_abs'] = sub(co_r.grad, 37)
    out['grad_pts_sub'], out['grad_pts_sum'], out['grad_pts_abs'] = sub(po_r.grad, 1)
    with torch.no_grad():
        rres = head.get_bboxes([rc], [rp], metas)
        dets, labs, keeps, cands, topks = [], [], [], [], []
        for b in range(len(metas)):
            ps, labels, al = op2p.get_bboxes_single(opd[b][..., :2], ocl[b], metas[b]['img_shape'], metas[b]['scale_factor'], cfg,
                                                    return_all=True)
            wh = torch.tensor(cfg['pseudo_wh'])
            eq(torch.cat([ps[:, :2] - wh / 2, ps[:, :2] + wh / 2, ps[:, 2:]], -1), rres[b][0], f'p2p defaults det[{b}]')
            eq(labels, rres[b][1], f'p2p defaults labels[{b}]')
            dets.append(rres[b][0]); labs.append(rres[b][1]); keeps.append(al['keep']); cands.append(al['cand_inds'])
            topks.append(al['topk_inds'])
    out['det_len'] = np.array([len(x) for x in dets])
    out['det'] = torch.cat(dets).numpy()
    out['det_labels'] = torch.cat(labs).numpy()
    out['keep'] = torch.cat(keeps).numpy()
    out['cand_len'] = np.array([len(x) for x in cands])
    out['topk'] = torch.cat(topks).numpy().astype(np.int32)
    out['seed'] = np.int64(seed)
    path = os.path.join(GOLD, 'p2p_defaults_lite.npz')
    np.savez_compressed(path, **out)
    print(f'[golden] {path}: {os.path.getsize(path) / 1024:.0f} KiB; dets/img {out["det_len"].tolist()} cands/img '
          f'{out["cand_len"].tolist()} pos {int((out["gt_inds"] > 0).sum())}; losses cls {out["loss_cls"].tolist()} pts {out["loss_pts"].tolist()}')


def main():
    torch.set_num_threads(os.cpu_count())
    os.makedirs(GOLD, exist_ok=True)
    golden_p2p_defaults(load_reference())


if __name__ == '__main__':
    main()
