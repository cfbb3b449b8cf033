"""Pins oracle/p2p_softmax.py against the REAL reference and writes tests/golden/p2p_softmax_lite.npz.  (test infrastructure)

Run in the build container only (needs /root/reference):   python -m oracle.make_golden_p2p_softmax
Same procedure and helpers as oracle/make_golden_p2p_defaults.py: the unmodified reference mmdet package is imported through
oracle/_mmcv_stub.py, two P2PHeads are built at the reference defaults (four point anchors per cell, MSELoss) with
  (a) CrossEntropyLoss(use_sigmoid=False, class_weight=[C+1 non-uniform values])  -> cls_out 4 x 81 = 324 channels
  (b) CrossEntropyLoss(use_sigmoid=True, class_weight=[C non-uniform values])     -> class_weight is binary_cross_entropy's pos_weight
reference and oracle run on the same seeded inputs and their equality is ASSERTED before the reference's outputs are stored.
The case is also asserted free of near-ties, so that the bit-exact comparisons of the CUDA path against the fixture are meaningful
although its softmax is not bit-identical to ATen's: no two keys among the top nms_pre + 1 within 1e-5 relative, no foreground
score of a top-k proposal within 1e-5 relative of score_thr, no two candidate scores within 1e-5 relative.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import p2p as op2p, p2p_softmax as osm  # noqa: E402
from oracle._mmcv_stub import load_reference, CfgDict  # noqa: E402
from oracle.make_golden import GOLD, eq, sub  # noqa: E402
from oracle.make_golden_p2p_defaults import P2P_DEFAULTS_TRAIN_CFG  # noqa: E402

SEED, NMS_PRE = 4267, 200
TEST_CFG = dict(nms_pre=NMS_PRE, min_bbox_size=0, score_thr=0.05, pseudo_wh=(32, 32), nms=dict(type='nms', iou_threshold=0.5),
                max_per_img=100)
TIE_REL = 1e-5


def class_weights(num_classes):
    """non-uniform class weights: (softmax C+1 values, sigmoid C values)."""
    sm = [round(0.5 + 0.01 * ((7 * c) % 101), 2) for c in range(num_classes)] + [0.75]
    sg = [round(2.0 - 0.015 * ((11 * c) % 97), 3) for c in range(num_classes)]
    return sm, sg


def min_rel_gap(v):
    v = torch.sort(v.double().flatten(), descending=True)[0]
    if len(v) < 2:
        return float('inf')
    return float(((v[:-1] - v[1:]) / v[:-1].abs()).min())


def build_head(HEADS, d, loss_cls):
    return HEADS.build(dict(type='P2PHead', num_classes=d['num_classes'], in_channels=d['C'], feat_channels=d['C'], stacked_convs=4,
                            strides=[d['stride']], norm_cfg=dict(type='GN', num_groups=32, requires_grad=True), loss_cls=loss_cls,
                            train_cfg=CfgDict(P2P_DEFAULTS_TRAIN_CFG), test_cfg=CfgDict(TEST_CFG)))


def loss_and_grads(head, rc, rp, inp, cfg, out, prefix):
    gtb, gtl, metas = inp['gt_bboxes'], inp['gt_labels'], inp['img_metas']
    with torch.no_grad():
        _, rpd, rv, rcl = head.get_pred_points([rc], [rp], metas)
        gt_points = head.pseudo_bbox_to_center(gtb)
        rl, rlw, rgp, rpw = head.get_targets(rpd[..., :2], rv, rcl, gt_points, gtl, metas, None)
        _, opd, ov, ocl = osm.pred_points(rc, rp, metas, cfg)
        tg = [op2p.target_single(opd[b][..., :2], ov[b], ocl[b], gt_points[b], gtl[b], metas[b]['img_shape'], cfg)
              for b in range(len(metas))]
        for b in range(len(metas)):
            eq(tg[b][0], rl[b], 'labels'); eq(tg[b][1], rlw[b], 'lw'); eq(tg[b][2], rgp[b], 'gpts'); eq(tg[b][3], rpw[b], 'pw')
    out[prefix + 'gt_inds'] = torch.stack([t[4] for t in tg]).numpy().astype(np.int32)
    out[prefix + 'labels'] = torch.stack([t[0] for t in tg]).numpy()
    co_r, po_r = rc.clone().requires_grad_(True), rp.clone().requires_grad_(True)
    rloss = head.loss([co_r], [po_r], gtb, gtl, metas, gt_bboxes_ignore=[torch.zeros(0, 4) for _ in metas])
    (sum(rloss['loss_cls']) + sum(rloss['loss_pts'])).backward()
    co, po = rc.clone().requires_grad_(True), rp.clone().requires_grad_(True)
    oloss = osm.p2p_loss(co, po, gtb, gtl, metas, cfg)
    (sum(oloss['loss_cls']) + sum(oloss['loss_pts'])).backward()
    for k in ('loss_cls', 'loss_pts'):
        eq(torch.stack(oloss[k]).detach(), torch.stack(rloss[k]).detach(), prefix + k, exact=False, tol=1e-6)
        out[prefix + k] = torch.stack(rloss[k]).detach().numpy()
    eq(co.grad, co_r.grad, prefix + 'dcls', exact=False, tol=1e-6)
    eq(po.grad, po_r.grad, prefix + 'dpts', exact=False, tol=1e-6)
    out[prefix + 'grad_cls_sub'], out[prefix + 'grad_cls_sum'], _ = sub(co_r.grad, 37)
    out[prefix + 'grad_pts_sub'], out[prefix + 'grad_pts_sum'], _ = sub(po_r.grad, 1)


def golden_p2p_softmax(HEADS, seed=SEED):
    import mmdet.models.point.dense_heads.p2p_head as ref_mod
    ref_mod.TestP2PHead.test_assign = staticmethod(lambda *a, **k: None)   # debug visualiser (needs huicv)
    inp = osm.inputs(seed)
    d = inp['cfgd']
    C = d['num_classes']
    cw_sm, cw_sg = class_weights(C)
    metas = inp['img_metas']
    out = {}
    # ---- (a) softmax CrossEntropyLoss with class_weight
    head = build_head(HEADS, d, dict(type='CrossEntropyLoss', use_sigmoid=False, class_weight=cw_sm, loss_weight=1.0))
    assert head.num_points == 4 and head.num_cls_out == C + 1 and head.cls_out.out_channels == 4 * (C + 1), head.cls_out
    head.load_state_dict(inp['weights'], strict=True)
    head.eval()
    cfg = osm.softmax_cfg(use_sigmoid=False, class_weight=cw_sm, num_classes=C, stride=d['stride'], nms_iou=0.5, nms_pre=NMS_PRE)
    with torch.no_grad():
        rc, rp = head((inp['x'],))
        rc, rp = rc[0], rp[0]
        oc, opo = op2p.head_forward(inp['x'], inp['weights'], cfg)
    eq(oc, rc, 'cls_out', exact=False, tol=1e-6)
    eq(opo, rp, 'pts_out', exact=False, tol=1e-6)
    out['cls_out_sub'], out['cls_out_sum'], out['cls_out_abs'] = sub(rc, 37)
    out['pts_out_sub'], out['pts_out_sum'], out['pts_out_abs'] = sub(rp, 1)
    loss_and_grads(head, rc, rp, inp, cfg, out, 'sm_')
    with torch.no_grad():
        rres = head.get_bboxes([rc], [rp], metas)
        _, opd, _, ocl = osm.pred_points(rc, rp, metas, cfg)
        dets, labs, keeps, cands, topks = [], [], [], [], []
        for b in range(len(metas)):
            ps, labels, al = osm.get_bboxes_single(opd[b][..., :2], ocl[b], metas[b]['img_shape'], metas[b]['scale_factor'], cfg,
                                                   return_all=True)
            wh = torch.tensor(cfg['pseudo_wh'])
            eq(torch.cat([ps[:, :2] - wh / 2, ps[:, :2] + wh / 2, ps[:, 2:]], -1), rres[b][0], f'softmax det[{b}]')
            eq(labels, rres[b][1], f'softmax labels[{b}]')
            # no near-ties: top-k boundary and order, the score_thr filter and the NMS order are decided with a margin
            top = torch.sort(al['keys'].double(), descending=True)[0][:NMS_PRE + 1]
            assert min_rel_gap(top) > TIE_REL, ('top-k near-tie', b, min_rel_gap(top))
            sc = al['scores'].double()
            assert float(((sc - cfg['score_thr']).abs() / cfg['score_thr']).min()) > TIE_REL, ('score_thr near-tie', b)
            assert min_rel_gap(sc[sc > cfg['score_thr']]) > TIE_REL, ('candidate near-tie', b)
            dets.append(rres[b][0]); labs.append(rres[b][1]); keeps.append(al['keep']); cands.append(al['cand_inds'])
            topks.append(al['topk_inds'])
    out['det_len'] = np.array([len(x) for x in dets])
    out['det'] = torch.cat(dets).numpy()
    out['det_labels'] = torch.cat(labs).numpy()
    out['keep'] = torch.cat(keeps).numpy()
    out['cand_len'] = np.array([len(x) for x in cands])
    out['topk'] = torch.cat(topks).numpy().astype(np.int32)
    # ---- (a) test-time augmentation in softmax mode: the reference's own aug_test_bboxes over prepared head outputs
    aug_outs, aug_metas = osm.aug_inputs(rc, rp, metas)
    table = {id(o[0]): o for o in aug_outs}
    head.forward = lambda x: ([table[id(x)][0]], [table[id(x)][1]])
    for rescale in (False, True):
        with torch.no_grad():
            rres = head.aug_test_bboxes([o[0] for o in aug_outs], aug_metas, rescale=rescale)
            ores, aux = osm.aug_test_bboxes(aug_outs, aug_metas, cfg, rescale=rescale)
        eq(ores[0][0], rres[0][0], f'aug det (rescale={rescale})')
        eq(ores[0][1], rres[0][1], f'aug labels (rescale={rescale})')
        assert len(rres[0][1]) > 0 and not bool((rres[0][1] == C - 1).any()), 'class C-1 is dropped by the softmax merge'
        # no near-ties in the merge either: between candidates of one class (suppression order) and among the kept scores (row order)
        ms = aux['merged_scores']
        assert all(min_rel_gap(ms[:, c][ms[:, c] > cfg['score_thr']]) > TIE_REL for c in range(C)), 'merge near-tie within a class'
        assert min_rel_gap(rres[0][0][:, 4]) > TIE_REL, 'near-tie among the merged detections'
        out[f'aug_det_rescale{int(rescale)}'] = rres[0][0].numpy()
        out[f'aug_labels_rescale{int(rescale)}'] = rres[0][1].numpy()
    for (c, p), m in zip(aug_outs, aug_metas):                 # every augmentation's own top-k / candidates free of near-ties
        _, apd, _, acl = osm.pred_points(c, p, m, cfg)
        _, _, al = osm.get_bboxes_single(apd[0][..., :2], acl[0], m[0]['img_shape'], m[0]['scale_factor'], cfg, return_all=True)
        sc = al['scores'].double()
        assert min_rel_gap(torch.sort(al['keys'].double(), descending=True)[0][:NMS_PRE + 1]) > TIE_REL, 'aug top-k near-tie'
        assert float(((sc - cfg['score_thr']).abs() / cfg['score_thr']).min()) > TIE_REL, 'aug score_thr near-tie'
        assert min_rel_gap(sc[sc > cfg['score_thr']]) > TIE_REL, 'aug candidate near-tie'
    per_aug_c1 = sum(int((osm.p2p_get_bboxes(c, p, m, cfg)[0][1] == C - 1).sum()) for (c, p), m in zip(aug_outs, aug_metas))
    assert per_aug_c1 > 0, 'the case must have per-aug detections of class C-1 for the merge to drop'
    out['aug_keep'] = aux['keep'].numpy()
    out['aug_n_merged'] = np.int64(len(aux['merged_boxes']))
    out['aug_per_aug_last_class'] = np.int64(per_aug_c1)
    # ---- (b) sigmoid CrossEntropyLoss with class_weight (= pos_weight) on the foreground columns of the same maps
    head_b = build_head(HEADS, d, dict(type='CrossEntropyLoss', use_sigmoid=True, class_weight=cw_sg, loss_weight=1.0))
    assert head_b.num_cls_out == C
    cfg_b = osm.softmax_cfg(use_sigmoid=True, class_weight=cw_sg, num_classes=C, stride=d['stride'], nms_iou=0.5, nms_pre=NMS_PRE)
    rc_b = rc.reshape(rc.shape[0], 4, C + 1, *rc.shape[2:])[:, :, :C].reshape(rc.shape[0], 4 * C, *rc.shape[2:]).contiguous()
    loss_and_grads(head_b, rc_b, rp, inp, cfg_b, out, 'sg_')
    out['class_weight_softmax'] = np.array(cw_sm, np.float32)
    out['class_weight_sigmoid'] = np.array(cw_sg, np.float32)
    out['seed'] = np.int64(seed)
    out['nms_pre'] = np.int64(NMS_PRE)
    path = os.path.join(GOLD, 'p2p_softmax_lite.npz')
    np.savez_compressed(path, **out)
    print(f'[golden] {path}: {os.path.getsize(path) / 1024:.0f} KiB; dets/img {out["det_len"].tolist()} cands/img '
          f'{out["cand_len"].tolist()} pos {int((out["sm_gt_inds"] > 0).sum())}; losses cls {out["sm_loss_cls"].tolist()} '
          f'pts {out["sm_loss_pts"].tolist()}; aug merged {int(out["aug_n_merged"])} -> {len(out["aug_keep"])} kept, '
          f'{per_aug_c1} per-aug detections of class {C - 1} dropped')


def main():
    torch.set_num_threads(os.cpu_count())
    os.makedirs(GOLD, exist_ok=True)
    golden_p2p_softmax(load_reference())


if __name__ == '__main__':
    main()
