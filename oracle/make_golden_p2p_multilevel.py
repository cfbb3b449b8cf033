"""Pins oracle/p2p_multilevel.py against the REAL reference and writes tests/golden/p2p_multilevel_*.npz.  (test infrastructure)

Run in the build container only (needs /root/reference):   python -m oracle.make_golden_p2p_multilevel
Same procedure and helpers as oracle/make_golden_p2p_defaults.py: the unmodified reference mmdet package is imported through
oracle/_mmcv_stub.py, a P2PHead with several strides is built for every case of oracle.p2p_multilevel.CASES, the reference and the
oracle run the same seeded weights and per-level feature maps (towers included), their equality is ASSERTED, then the reference's
losses, parameter gradients (strided samples + float64 sums), assignments, targets, per-chunk top-k indices, NMS keep and
detections are stored.  Case d_uneven stores training only and asserts that the reference's inference raises.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import p2p_multilevel as oml  # noqa: E402
from oracle._mmcv_stub import load_reference, CfgDict  # noqa: E402
from oracle.make_golden import GOLD, eq, sub  # noqa: E402
from oracle.make_golden_p2p_defaults import P2P_DEFAULTS_TRAIN_CFG  # noqa: E402

GRAD_STEP = 97        # strided sample of every conv weight gradient; biases and GroupNorm parameters are stored whole


def test_cfg(cfg):
    return dict(nms_pre=cfg['nms_pre'], min_bbox_size=0, score_thr=0.05, pseudo_wh=(32, 32), nms=dict(type='nms', iou_threshold=0.5),
                max_per_img=100)


def build_head(HEADS, cfg):
    import mmdet.models.point.dense_heads.p2p_head as ref_mod
    ref_mod.TestP2PHead.test_assign = staticmethod(lambda *a, **k: None)   # debug visualiser (needs huicv)
    if cfg['loss_cls'] == 'FocalLoss':
        loss_cls = dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=cfg['loss_cls_weight'])
    else:
        loss_cls = dict(type='CrossEntropyLoss', use_sigmoid=cfg.get('use_sigmoid', True), loss_weight=cfg['loss_cls_weight'],
                        class_weight=cfg.get('class_weight'))
    if cfg['loss_reg'] == 'SmoothL1Loss':
        loss_reg = dict(type='SmoothL1Loss', beta=cfg['sl1_beta'], loss_weight=cfg['loss_reg_weight'])
    else:
        loss_reg = dict(type='MSELoss', loss_weight=cfg['loss_reg_weight'])
    return HEADS.build(dict(type='P2PHead', num_classes=cfg['num_classes'], in_channels=oml.C_FEAT, feat_channels=oml.C_FEAT,
                            stacked_convs=4, strides=list(cfg['strides']), point_anchor=[tuple(a) for a in cfg['point_anchor']],
                            pts_gamma=cfg['pts_gamma'], reg_norm=cfg['reg_norm'], loss_cls=loss_cls, loss_reg=loss_reg,
                            norm_cfg=dict(type='GN', num_groups=32, requires_grad=True), train_cfg=CfgDict(P2P_DEFAULTS_TRAIN_CFG),
                            test_cfg=CfgDict(test_cfg(cfg))))


def golden_case(HEADS, name):
    inp, cfg = oml.case_inputs(name)
    head = build_head(HEADS, cfg)
    head.load_state_dict(inp['weights'], strict=True)
    gtb, gtl, metas = inp['gt_bboxes'], inp['gt_labels'], inp['img_metas']
    out = dict(seed=np.int64(oml.CASES[name]['seed']))
    # training: the reference head end to end, parameter gradients
    head.train()
    head.zero_grad()
    rc, rp = head(inp['xs'])
    rloss = head.loss(rc, rp, gtb, gtl, metas, gt_bboxes_ignore=[torch.zeros(0, 4) for _ in metas])
    (sum(rloss['loss_cls']) + sum(rloss['loss_pts'])).backward()
    w = {k: v.clone().requires_grad_(True) for k, v in inp['weights'].items()}
    oc, opo = oml.head_forward(inp['xs'], w, cfg)
    for l in range(len(rc)):
        eq(oc[l], rc[l].detach(), f'{name} cls_out[{l}]', exact=False, tol=1e-6)
        eq(opo[l], rp[l].detach(), f'{name} pts_out[{l}]', exact=False, tol=1e-6)
    oloss, aux = oml.p2p_loss(oc, opo, gtb, gtl, metas, cfg, return_all=True)
    (sum(oloss['loss_cls']) + sum(oloss['loss_pts'])).backward()
    for k in ('loss_cls', 'loss_pts'):
        eq(torch.stack(oloss[k]).detach(), torch.stack(rloss[k]).detach(), f'{name} {k}', exact=False, tol=1e-6)
        out[k] = torch.stack(rloss[k]).detach().numpy()
    params = dict(head.named_parameters())
    for k, v in w.items():
        eq(v.grad, params[k].grad, f'{name} d/d{k}', exact=False, tol=1e-5)
        step = GRAD_STEP if v.dim() == 4 else 1
        out[f'grad/{k}'], out[f'gradsum/{k}'], _ = sub(params[k].grad, step)
    with torch.no_grad():
        _, rpd, rv, rcl = head.get_pred_points([c.detach() for c in rc], [p.detach() for p in rp], metas)
        rl, rlw, rgp, rpw = head.get_targets(rpd[..., :2], rv, rcl, head.pseudo_bbox_to_center(gtb), gtl, metas, None)
    tg = aux['targets']
    for b in range(len(metas)):
        eq(tg[b][0], rl[b], 'labels'); eq(tg[b][1], rlw[b], 'lw'); eq(tg[b][2], rgp[b], 'gpts'); eq(tg[b][3], rpw[b], 'pw')
    out['gt_inds'] = torch.stack([t[4] for t in tg]).numpy().astype(np.int32)
    out['labels'] = torch.stack(rl).numpy()
    out['gt_pts'] = torch.stack(rgp).numpy()
    # inference
    head.eval()
    with torch.no_grad():
        rc, rp = head(inp['xs'])
        oc, opo = oml.head_forward(inp['xs'], inp['weights'], cfg)
        for l in range(len(rc)):      # the GPU tests feed the oracle's maps to the CUDA get_bboxes in place of these
            eq(oc[l], rc[l], f'{name} eval cls_out[{l}]')
            eq(opo[l], rp[l], f'{name} eval pts_out[{l}]')
        T = sum(c.shape[-2] * c.shape[-1] for c in rc) * len(cfg['point_anchor'])
        out['T'] = np.int64(T)
        if T % len(rc):
            try:
                head.get_bboxes(rc, rp, metas)
            except RuntimeError as e:
                out['ref_error'] = np.array(str(e))
            else:
                raise AssertionError(f'{name}: the reference accepted T % L != 0')
        else:
            rres = head.get_bboxes(rc, rp, metas)
            ores, oaux = oml.p2p_get_bboxes(rc, rp, metas, cfg, return_all=True)
            for b in range(len(metas)):
                eq(ores[b][0], rres[b][0], f'{name} det[{b}]', exact=False, tol=1e-6)
                eq(ores[b][1], rres[b][1], f'{name} labels[{b}]')
            out['det_len'] = np.array([len(r[0]) for r in rres])
            out['det'] = torch.cat([r[0] for r in rres]).numpy()
            out['det_labels'] = torch.cat([r[1] for r in rres]).numpy()
            out['keep'] = torch.cat([a['keep'] for a in oaux]).numpy()
            out['topk'] = torch.stack([torch.stack(a['topk_inds']) for a in oaux]).numpy().astype(np.int32)
    path = os.path.join(GOLD, f'p2p_multilevel_{name}.npz')
    np.savez_compressed(path, **out)
    print(f'[golden] {path}: {os.path.getsize(path) / 1024:.0f} KiB; T {T}; pos {int((out["gt_inds"] > 0).sum())}; '
          f'dets/img {out.get("det_len", np.array([])).tolist()}; losses cls {out["loss_cls"].tolist()} pts {out["loss_pts"].tolist()}')


def golden_aug(HEADS):
    feats, metas, w, cfg = oml.aug_inputs()
    head = build_head(HEADS, cfg)
    head.load_state_dict(w, strict=True)
    head.eval()
    with torch.no_grad():
        rres = head.aug_test_bboxes(feats, metas, rescale=False)
        outs = [head(x) for x in feats]
        ores, _ = oml.aug_test_bboxes(outs, metas, cfg)
    eq(ores[0][0], rres[0][0], 'aug det', exact=False, tol=1e-6)
    eq(ores[0][1], rres[0][1], 'aug labels')
    path = os.path.join(GOLD, 'p2p_multilevel_aug.npz')
    np.savez_compressed(path, det=rres[0][0].numpy(), det_labels=rres[0][1].numpy(), seed=np.int64(oml.AUG_CASE['seed']))
    print(f'[golden] {path}: {len(rres[0][0])} merged detections')


def main():
    torch.set_num_threads(os.cpu_count())
    os.makedirs(GOLD, exist_ok=True)
    HEADS = load_reference()
    for name in oml.CASES:
        golden_case(HEADS, name)
    golden_aug(HEADS)


if __name__ == '__main__':
    main()
