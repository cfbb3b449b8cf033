"""Pins oracle/p2p_loss_types.py against the REAL reference and writes tests/golden/p2p_loss_types_*.npz.  (test infrastructure)

Run in the build container only (needs /root/reference):   python -m oracle.make_golden_p2p_loss_types
Same procedure as oracle/make_golden_p2p_multilevel.py: the unmodified reference mmdet package is imported through oracle/_mmcv_stub.py,
a P2PHead is built with the case's loss_cls / loss_reg for every case of oracle.p2p_loss_types.CASES and trained for the case's steps
(the same head, so GHM's acc_sum carries over), the oracle runs the same seeded weights and feature maps, and their agreement is
ASSERTED: output maps and acc_sum bit-equal, losses and gradients within 1e-6, every GHMR g at least SAFE_MARGIN from a bin edge.  Stored
per step: the losses, acc_sum, the oracle's per-image bin counts and margins; for the last step: the gradients of the output maps
(whole) and of the parameters (strided samples), the targets, and the reference head's state_dict names and shapes.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import p2p_loss_types as olt, p2p_multilevel as oml  # noqa: E402
from oracle._mmcv_stub import load_reference, CfgDict  # noqa: E402
from oracle.make_golden import GOLD, eq, sub  # noqa: E402
from oracle.make_golden_p2p_defaults import P2P_DEFAULTS_TRAIN_CFG  # noqa: E402

GRAD_STEP = 97


def head_kwargs(cfg):
    """the P2PHead constructor arguments of a case, shared by the reference build here and the CUDA head in tests/."""
    return dict(num_classes=cfg['num_classes'], in_channels=olt.C_FEAT, feat_channels=olt.C_FEAT, stacked_convs=4,
                strides=list(cfg['strides']), point_anchor=[tuple(a) for a in cfg['point_anchor']], pts_gamma=cfg['pts_gamma'],
                reg_norm=cfg['reg_norm'], loss_cls=dict(cfg['loss_cls_cfg']), loss_reg=dict(cfg['loss_reg_cfg']),
                norm_cfg=dict(type='GN', num_groups=32, requires_grad=True))


def build_head(HEADS, cfg):
    import mmdet.models.point.dense_heads.p2p_head as ref_mod
    ref_mod.TestP2PHead.test_assign = staticmethod(lambda *a, **k: None)   # debug visualiser (needs huicv)
    return HEADS.build(dict(type='P2PHead', **head_kwargs(cfg), train_cfg=CfgDict(P2P_DEFAULTS_TRAIN_CFG),
                            test_cfg=CfgDict(nms_pre=100, min_bbox_size=0, score_thr=0.05, pseudo_wh=(32, 32),
                                             nms=dict(type='nms', iou_threshold=0.5), max_per_img=100)))


def golden_case(HEADS, name):
    c = olt.CASES[name]
    inp, cfg = olt.case_inputs(name)
    head = build_head(HEADS, cfg)
    state = olt.make_state(cfg)
    sd = dict(inp['weights'], **{k: v.clone() for k, v in state.items()})
    head.load_state_dict(sd, strict=True)
    rsd = head.state_dict()
    out = dict(seed=np.int64(c['seed']), state_keys=np.array(sorted(rsd)),
               state_shapes=np.array([list(rsd[k].shape) + [-1] * (4 - rsd[k].dim()) for k in sorted(rsd)], np.int64))
    for k in state:
        out[f'edges_init/{k}'] = rsd[k].numpy().copy()
    steps = c.get('steps', 1)
    for step in range(steps):
        inp, _ = olt.case_inputs(name, step)
        gtb, gtl, metas = inp['gt_bboxes'], inp['gt_labels'], inp['img_metas']
        head.train()
        head.zero_grad()
        rc, rp = head(inp['xs'])
        for t in rc + rp:
            t.retain_grad()
        rloss = head.loss(rc, rp, gtb, gtl, metas, gt_bboxes_ignore=[torch.zeros(0, 4) for _ in metas])
        (sum(rloss['loss_cls']) + sum(rloss['loss_pts'])).backward()
        w = {k: v.clone().requires_grad_(True) for k, v in inp['weights'].items()}
        oc, opo = oml.head_forward(inp['xs'], w, cfg)
        for l in range(len(rc)):
            eq(oc[l], rc[l].detach(), f'{name} cls_out[{l}]')       # bit-equal: the GPU tests feed the oracle's maps to the loss
            eq(opo[l], rp[l].detach(), f'{name} pts_out[{l}]')
        oloss, aux = olt.p2p_loss(oc, opo, gtb, gtl, metas, cfg, state, return_all=True)
        (sum(oloss['loss_cls']) + sum(oloss['loss_pts'])).backward()
        for k in ('loss_cls', 'loss_pts'):
            r = torch.stack([v.reshape(()) for v in rloss[k]]).detach()
            eq(torch.stack([v.reshape(()) for v in oloss[k]]).detach(), r, f'{name} step {step} {k}', exact=False, tol=1e-6)
            out[f'{k}/{step}'] = r.numpy()
        for k, v in state.items():
            if k.endswith('acc_sum'):
                eq(v, head.state_dict()[k], f'{name} step {step} {k}')          # bit-equal
                out[f'{k}/{step}'] = v.numpy().copy()
        for kind in ('cls', 'reg'):
            if aux[f'{kind}_counts']:
                out[f'{kind}_counts/{step}'] = torch.stack(aux[f'{kind}_counts']).numpy().astype(np.int32)
                mg = min(aux[f'{kind}_margin'])
                out[f'{kind}_margin/{step}'] = np.float64(mg)
                assert kind == 'cls' or mg >= olt.SAFE_MARGIN, f'{name} step {step}: a {kind} g lies {mg:.2e} from a bin edge'
        if step == steps - 1:
            params = dict(head.named_parameters())
            for k, v in w.items():
                eq(v.grad, params[k].grad, f'{name} d/d{k}', exact=False, tol=1e-5)
                out[f'grad/{k}'] = sub(params[k].grad, GRAD_STEP if v.dim() == 4 else 1)[0]
            for l in range(len(rc)):
                out[f'dmap_cls/{l}'] = rc[l].grad.numpy()
                out[f'dmap_pts/{l}'] = rp[l].grad.numpy()
            tg = aux['targets']
            out['gt_inds'] = torch.stack([t[4] for t in tg]).numpy().astype(np.int32)
            out['labels'] = torch.stack([t[0] for t in tg]).numpy()
    path = os.path.join(GOLD, f'p2p_loss_types_{name}.npz')
    np.savez_compressed(path, **out)
    margins = {k: float(v) for k, v in out.items() if 'margin' in k}
    print(f'[golden] {path}: {os.path.getsize(path) / 1024:.0f} KiB; pos {int((out["gt_inds"] > 0).sum())}; '
          f'losses cls {out[f"loss_cls/{steps - 1}"].tolist()} pts {out[f"loss_pts/{steps - 1}"].tolist()}; margins {margins}')


def main():
    torch.set_num_threads(os.cpu_count())
    os.makedirs(GOLD, exist_ok=True)
    HEADS = load_reference()
    for name in (sys.argv[1:] or olt.CASES):
        golden_case(HEADS, name)


if __name__ == '__main__':
    main()
