"""Parity on the EXACT shapes the metric is quoted on (VERDICT r1 item 1; BASELINE.json configs[1], [2], [4]) plus
P2PHead.aug_test_bboxes.

* config 2 (B=8, 100x168x256 map, 500 points / image, r=8): the PRODUCT step the bench times — wgmma towers -> 1-tap logit conv ->
  ptb_cpr_refine_fused — for all 8 images against oracle tower_forward + cpr_get_bboxes, through the float64 decision-margin harness
  of tests/helpers.py (SURVEY.md §7.1): every chosen-mask / not_refine decision with margin > bound is bit-equal, floats 1e-4.
* config 5 shard shape (2000 points / image): same harness on image 0 (replaces round 1's "<= 3 rows may differ" allowance).
* config 3 (B=16, 16 800 proposals / image): P2PHead post-processing bit-exact (top-k indices, NMS keep) at iou 0.01 and 0.5; the
  full oracle (global class-offset NMS, ~10 s / image on the host) on 3 images, the exact per-class replay on all 16.
* aug_test_bboxes with flip + scale + tile_offset against the oracle restatement and the reference-pinned golden vectors.
"""
import os

import numpy as np
import pytest
import torch

from oracle import cpr as ocpr, p2p as op2p, synth
from tests.helpers import assert_close, assert_mask_equal, check_refine_against_oracle, nms_replay_per_class, oracle_cfg
from tests.test_gpu_cpr_head import head_cfg

pytestmark = pytest.mark.gpu


def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')


def _build_cpr(inp, weights):
    from pointtinybenchmark_b200 import cpr_head  # noqa: F401
    from pointtinybenchmark_b200.registry import build_head
    head = build_head(head_cfg(inp['cfgd'])).cuda().eval()
    sd = head.state_dict()
    sd.update(weights)
    head.load_state_dict(sd, strict=True)
    return head


def _cat_refine(allo):
    ora = {k: torch.cat([r[k] for r in allo['refine']]) for k in allo['refine'][0]}
    ora['mask_valid'] = allo['ex']['pos_valid'][:, 0, :, 0]
    return ora


@pytest.fixture(scope='module')
def config2():
    """headline inputs + the oracle's tower output (computed once: 634 GFLOP of fp32 conv on the host)."""
    _need_cuda()
    inp = synth.cpr_inputs('headline', 2024, trained_like=False, with_towers=True)
    cfg = oracle_cfg(inp['cfgd'])
    with torch.no_grad():
        feat_o = ocpr.tower_forward(inp['cls_feat'], inp['weights'], cfg)
    return inp, cfg, feat_o


@pytest.mark.parametrize('variant', ['bench_weights', 'spread'])
def test_config2_full_shape_product_step_and_pieces_vs_oracle(config2, variant):
    from pointtinybenchmark_b200 import ops
    from pointtinybenchmark_b200.cpr_head import _BatchGT
    from pointtinybenchmark_b200.layers import tower, _packed_tc
    dev = torch.device('cuda:0')
    inp, cfg, feat_o = config2
    w = dict(inp['weights'])
    g = torch.Generator().manual_seed(5)
    if variant == 'bench_weights':          # bench.py::head_weights(): Normal(0, 0.08) classifier, bias -log(99)
        w['cls_out.weight'] = torch.randn(80, 256, generator=g) * 0.08
    else:                                   # probabilities spread over (0, 1): every filter of the refiner has work to do
        w['cls_out.weight'] = torch.randn(80, 256, generator=g) * 0.16
        w['cls_out.bias'] = torch.full((80,), -2.0)
    head = _build_cpr(inp, w)
    gtb = [b.to(dev) for b in inp['gt_bboxes']]
    gtl = [l.to(dev) for l in inp['gt_labels']]
    aid = [a.to(dev) for a in inp['gt_anns_id']]
    x = inp['cls_feat'].to(dev)
    metas = inp['img_metas']
    # ---- the product call (what bench.py times)
    with torch.no_grad():
        res = head.simple_test((x,), metas, gt_bboxes=gtb, gt_labels=gtl, gt_anns_id=aid)
        assert head.last_tower_backend == 'wgmma-f16x2'
        # the same step in pieces, to look inside: fp16 pair of the tower output -> logit map -> fused refine with the chosen mask
        info = {}
        h, l = tower(head.cls_convs, x, info, want='f16pair')
        lmap = ops.conv_tc_f16(h, l, _packed_tc(head.cls_out, 1), 1, head.num_classes, bias=head.cls_out.bias.detach())
        gt = _BatchGT(gtb, gtl, metas, dev)
        got = head._refine_from_logit_map(lmap, gt, want_chosen=True)
        feat_g = head((x,))[0][0]
    det_pieces = torch.cat([got[0] - 8.0, got[0] + 8.0, got[1][:, None]], 1)
    assert torch.equal(torch.cat([r[0] for r in res])[:, :5], det_pieces), 'simple_test == its pieces (deterministic)'
    # ---- oracle: reference data flow on the host (gather 256 channels, Linear per sample)
    e_t = assert_close(feat_g, feat_o, 1e-4, 'wgmma towers vs oracle tower_forward at 8x256x100x168')
    with torch.no_grad():
        ores, allo = ocpr.cpr_get_bboxes(feat_o, w, inp['gt_bboxes'], inp['gt_labels'], inp['gt_anns_id'], metas, cfg, return_all=True)
    ora = _cat_refine(allo)
    prob_o = allo['bag_prob'][:, 0]                                      # (G,K,C)
    off = head._offsets(head.refine_pts_extractor['pos_generator'], dev)
    bl, _, valid = ops.bag_gather(lmap, gt.centers, gt.bag_img, off, head.strides[0], gt.pad_hw, pts=False)
    prob_g = torch.sigmoid(bl[..., :head.num_classes]).cpu()
    assert_mask_equal(valid, ora['mask_valid'], 'pos_valid at the headline shape')
    delta = float((prob_g.double() - prob_o.double()).abs().max())
    e_p = assert_close(prob_g, prob_o, 1e-4, 'bag probabilities of the product path vs oracle')
    bound = max(1e-5, 2.0 * delta)
    labels = torch.cat(inp['gt_labels'])
    stats = check_refine_against_oracle(got, ora, prob_o, labels, cfg, bound, f'config 2 [{variant}]')
    print(f'[config 2 {variant}] tower err {e_t:.1e}, prob err {e_p:.1e} (max |dp| {delta:.2e}), not_refine frac '
          f'{float(ora["not_refine"].float().mean()):.3f}, chosen / bag {float(ora["chosen"].float().sum(1).mean()):.1f}')
    assert stats['within_bound'] <= 2e-3 * stats['samples'], 'the within-bound set must stay small (bench weights: 80 near-equal class probabilities)'
    # output rows: everything but the (reported) within-bound GTs agrees with the oracle's get_bboxes
    det_o = torch.cat([r[0] for r in ores])
    flips = (got[3].cpu().bool() != ora['chosen'].bool()).any(dim=1) | (got[2].cpu().bool() != ora['not_refine'].bool())
    assert_close(torch.cat([r[0] for r in res]).cpu()[~flips][:, :5], det_o[~flips][:, :5], 1e-4, 'det rows vs oracle get_bboxes')
    assert torch.equal(torch.cat([r[0] for r in res]).cpu()[:, 5], det_o[:, 5]), 'ann ids'


def test_config2_full_shape_point_path_planted_evidence():
    """same shape, the point path alone on a feature map with class evidence planted around 80 % of the GTs (oracle/synth.py): ~20 chosen
    samples per bag, ~19 % not_refine — every filter of PointRefiner works.  CPRHead.get_bboxes (fp32 FFMA logit map + fused refine)
    vs the oracle's reference data flow, bound 1e-5 on the probabilities."""
    _need_cuda()
    dev = torch.device('cuda:0')
    inp = synth.cpr_inputs('headline', 2025)
    cfg = oracle_cfg(inp['cfgd'])
    head = _build_cpr(inp, inp['weights'])
    from pointtinybenchmark_b200.cpr_head import _BatchGT
    gtb = [b.to(dev) for b in inp['gt_bboxes']]
    gtl = [l.to(dev) for l in inp['gt_labels']]
    aid = [a.to(dev) for a in inp['gt_anns_id']]
    gt = _BatchGT(gtb, gtl, inp['img_metas'], dev)
    feat = inp['cls_feat'].to(dev)
    got = head.refine_points(feat, gt, want_chosen=True)
    res = head.get_bboxes([feat], [feat], inp['img_metas'], gt_bboxes=gtb, gt_labels=gtl, gt_anns_id=aid)
    with torch.no_grad():
        ores, allo = ocpr.cpr_get_bboxes(inp['cls_feat'], inp['weights'], inp['gt_bboxes'], inp['gt_labels'], inp['gt_anns_id'],
                                         inp['img_metas'], cfg, return_all=True)
    ora = _cat_refine(allo)
    stats = check_refine_against_oracle(got, ora, allo['bag_prob'][:, 0], torch.cat(inp['gt_labels']), cfg, 1e-5,
                                        'config 2, point path, planted evidence')
    assert stats['within_bound'] <= 1e-3 * stats['samples']
    assert 0.05 < float(ora['not_refine'].float().mean()) < 0.6 and float(ora['chosen'].float().sum(1).mean()) > 5
    flips = (got[3].cpu().bool() != ora['chosen'].bool()).any(dim=1) | (got[2].cpu().bool() != ora['not_refine'].bool())
    det, det_o = torch.cat([r[0] for r in res]).cpu(), torch.cat([r[0] for r in ores])
    assert_close(det[~flips][:, :5], det_o[~flips][:, :5], 1e-4, 'det rows vs oracle get_bboxes')
    assert torch.equal(det[:, 5], det_o[:, 5]), 'ann ids'


def test_config5_shape_margin_harness():
    """BASELINE.json configs[4] per-GPU shard shape (2000 points / image = 578 k bag samples): image 0 against the oracle through the
    margin harness (bound 1e-5 on the probabilities)."""
    _need_cuda()
    dev = torch.device('cuda:0')
    inp = synth.cpr_inputs('cpr2000', 31, B=1)
    cfg = oracle_cfg(inp['cfgd'])
    head = _build_cpr(inp, inp['weights'])
    from pointtinybenchmark_b200.cpr_head import _BatchGT
    gtb = [b.to(dev) for b in inp['gt_bboxes']]
    gtl = [l.to(dev) for l in inp['gt_labels']]
    gt = _BatchGT(gtb, gtl, inp['img_metas'], dev)
    got = head.refine_points(inp['cls_feat'].to(dev), gt, want_chosen=True)
    with torch.no_grad():
        _, allo = ocpr.cpr_get_bboxes(inp['cls_feat'], inp['weights'], inp['gt_bboxes'], inp['gt_labels'], inp['gt_anns_id'],
                                      inp['img_metas'], cfg, return_all=True)
    stats = check_refine_against_oracle(got, _cat_refine(allo), allo['bag_prob'][:, 0], torch.cat(inp['gt_labels']), cfg, 1e-5,
                                        'config 5 shard shape')
    assert stats['within_bound'] <= 1e-3 * stats['samples']


# ---------------------------------------------------------------------------------------------------------------------------------
def _p2p_head(d, iou, **over):
    from pointtinybenchmark_b200 import p2p_head  # noqa: F401
    from pointtinybenchmark_b200.registry import build_head
    from tests.test_gpu_p2p import head_cfg as p2p_cfg
    c = p2p_cfg(d, iou)
    c.update(over)
    return build_head(c).cuda().eval()


@pytest.mark.parametrize('iou', [0.01, 0.5])
def test_config3_full_shape_topk_and_nms_bit_exact(iou):
    """16 images x 16 800 proposals x 80 classes, nms_pre 1000, score_thr 0.05, max 100 (p2p_head.py:345-423, bbox_nms.py:7-94)."""
    _need_cuda()
    dev = torch.device('cuda:0')
    inp = synth.p2p_inputs('headline', 4321)
    d = inp['cfgd']
    assert inp['cls_out'].shape == (16, 80, 100, 168)
    cfg = op2p.default_cfg(num_classes=d['num_classes'], stride=d['stride'], nms_iou=iou)
    head = _p2p_head(d, iou)
    res, aux = head.get_bboxes([inp['cls_out'].to(dev)], [inp['pts_out'].to(dev)], inp['img_metas'], return_all=True)
    _, pred, _, cls = op2p.pred_points(inp['cls_out'], inp['pts_out'], inp['img_metas'], cfg)
    full = (0, 7, 15)
    wh = torch.tensor(cfg['pseudo_wh'])
    n_tied = 0
    for b, m in enumerate(inp['img_metas']):
        scores = cls[b].sigmoid()
        keys = scores.max(dim=1)[0]
        _, topk = keys.topk(cfg['nms_pre'])
        got = aux['topk_idx'][b].cpu().long()
        # torch.topk gives no order contract inside a group of EXACTLY equal keys (1000 fp32 keys in [0.87, 1): an exact tie in ~20 % of
        # the images); everything else must be bit-equal: same keys position by position, same set, same order outside tie groups
        assert torch.equal(keys[got], keys[topk]), f'top-k keys, image {b}'
        assert torch.equal(torch.sort(got)[0], torch.sort(topk)[0]), f'top-k set, image {b}'
        diff = got != topk
        if bool(diff.any()):
            kd = keys[topk][diff]
            assert all(int((keys[topk] == v).sum()) >= 2 for v in kd.tolist()), f'top-k order differs outside a tie group, image {b}'
            n_tied += int(diff.sum())
        n = int(aux['count'][b])
        # post-processing on the kernel's own (tie-equivalent) order: candidates in (position, class) order like multiclass_nms
        pts = pred[b][got][..., :2]
        pts = torch.stack([pts[:, 0].clamp(0, m['img_shape'][1]), pts[:, 1].clamp(0, m['img_shape'][0])], -1)
        sc_sel = scores[got]
        boxes_all = torch.cat([pts - wh / 2, pts + wh / 2], -1)
        if b in full:       # the oracle's global class-offset NMS (bbox_nms.py:7-94 + mmcv batched_nms)
            dets, labels, keep_o, inds = op2p.multiclass_nms(boxes_all, torch.cat([sc_sel, sc_sel.new_zeros(len(sc_sel), 1)], 1),
                                                             cfg['score_thr'], iou, cfg['max_per_img'])
            assert int(aux['cand_count'][b]) == len(inds)
            assert n == len(keep_o) and torch.equal(aux['keep'][b, :n].cpu().long(), keep_o), f'NMS keep, image {b}'
            assert torch.equal(res[b][1].cpu(), labels)
            cxcy = torch.stack([(dets[:, 0] + dets[:, 2]) / 2, (dets[:, 1] + dets[:, 3]) / 2], -1)
            assert_close(res[b][0], torch.cat([cxcy - wh / 2, cxcy + wh / 2, dets[:, 4:5]], -1), 1e-4, f'boxes, image {b}')
        # exact per-class replay (all images)
        sc = sc_sel.reshape(-1)
        cand = torch.nonzero(sc > cfg['score_thr']).squeeze(1)
        keep = nms_replay_per_class(boxes_all[cand // 80].numpy(), sc[cand].numpy(), (cand % 80).numpy(), iou, cfg['max_per_img'])
        assert int(aux['cand_count'][b]) == len(cand)
        assert n == len(keep) and np.array_equal(aux['keep'][b, :n].cpu().numpy().astype(np.int64), keep), f'per-class replay, image {b}'
    print(f'[config 3, iou {iou}] top-k positions permuted inside exact-tie groups: {n_tied}')
    print(f'[config 3, iou {iou}] candidates / image {aux["cand_count"].cpu().tolist()[:4]}..., kept {aux["count"].cpu().tolist()[:4]}...')


def test_config3_simple_test_through_the_towers():
    """P2PHead.simple_test at 16 x (256,100,168): forward (two wgmma towers + conv3x3 outputs) within 1e-4 of the oracle on two
    images; post-processing bit-exact on the head's OWN outputs for all 16 (top-k) / 2 images (full oracle NMS)."""
    _need_cuda()
    dev = torch.device('cuda:0')
    d = dict(synth.P2P_CONFIGS['headline'])
    g = torch.Generator().manual_seed(77)
    head = _p2p_head(d, 0.5)
    with torch.no_grad():
        head.cls_out.weight.mul_(4.4)                  # trained-like spread: logit std ~1.5 around the -log(99) bias
    head.cls_out.weight._version  # noqa: B018 (in-place mul_ above bumps the version: packed caches repack)
    x = torch.randn(16, 256, 100, 168, generator=g)
    metas = [dict(pad_shape=d['pad_hw'] + (3,), img_shape=d['img_hw'] + (3,), scale_factor=[1.0, 1.0, 1.0, 1.0])] * 16
    with torch.no_grad():
        cls_outs, pts_outs = head.forward((x.to(dev),))
        res, aux = head.get_bboxes(cls_outs, pts_outs, metas, return_all=True)
        res2 = head.simple_test((x.to(dev),), metas)
    for a, b in zip(res, res2):
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    cfg = op2p.default_cfg(num_classes=d['num_classes'], stride=d['stride'], nms_iou=0.5)
    w = {k: v.detach().cpu() for k, v in head.state_dict().items()}
    with torch.no_grad():
        oc, op_ = op2p.head_forward(x[:2], w, cfg)
    assert_close(cls_outs[0][:2], oc, 1e-4, 'cls_out through the towers')
    assert_close(pts_outs[0][:2], op_, 1e-4, 'pts_out through the towers')
    co, po = cls_outs[0].float().cpu().contiguous(), pts_outs[0].float().cpu().contiguous()
    _, pred, _, cls = op2p.pred_points(co, po, metas, cfg)
    for b in range(16):
        keys = cls[b].sigmoid().max(dim=1)[0]
        _, topk = keys.topk(cfg['nms_pre'])
        got = aux['topk_idx'][b].cpu().long()
        # sigmoid is bit-identical to ATen's CPU kernel, so the keys are too; only the order inside exact-tie groups is free
        assert torch.equal(keys[got], keys[topk]) and torch.equal(torch.sort(got)[0], torch.sort(topk)[0]), f'top-k, image {b}'
    for b in (0, 9):
        ps, labels, al = op2p.get_bboxes_single(pred[b][..., :2], cls[b], metas[b]['img_shape'], metas[b]['scale_factor'], cfg,
                                                return_all=True)
        n = int(aux['count'][b])
        assert n == len(al['keep'])
        assert torch.equal(res[b][1].cpu(), labels), f'labels of the kept detections, image {b}'
        assert_close(res[b][0][:, :4], torch.cat([ps[:, :2] - 16, ps[:, :2] + 16], -1), 1e-4, f'kept boxes, image {b}')


# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name,seed,iou', [('lite', 2468, 0.5), ('mid', 1357, 0.3)])
def test_aug_test_bboxes_flip_scale_tile_offset(golden_dir, name, seed, iou):
    """P2PHead.aug_test_bboxes (p2p_head.py:487-572 + dense_test_mixins.py:173-204 + transforms.py:62-85): per-aug NMS, score scatter,
    mapping back with flip / scale_factor / tile_offset, second multiclass NMS.  `forward` returns prepared head outputs on both sides."""
    _need_cuda()
    dev = torch.device('cuda:0')
    inp = synth.p2p_aug_inputs(name, seed)
    d = inp['cfgd']
    cfg = op2p.default_cfg(num_classes=d['num_classes'], stride=d['stride'], nms_iou=iou)
    gold = np.load(os.path.join(golden_dir, f'p2p_aug_{name}.npz'))
    head = _p2p_head(d, iou)
    dev_outs = [(c.to(dev), p.to(dev)) for c, p in inp['outs']]
    table = {id(o[0]): o for o in dev_outs}
    head.forward = lambda x: ([table[id(x)][0]], [table[id(x)][1]])
    for rescale in (False, True):
        res = head.aug_test_bboxes([o[0] for o in dev_outs], inp['metas'], rescale=rescale)
        ores, aux = op2p.aug_test_bboxes(inp['outs'], inp['metas'], cfg, rescale=rescale)
        assert len(res) == 1
        det, lab = res[0][0].cpu(), res[0][1].cpu()
        assert det.shape == ores[0][0].shape
        assert torch.equal(lab, ores[0][1]), 'labels after the second NMS'
        assert np.array_equal(lab.numpy(), gold[f'labels_rescale{int(rescale)}'])
        assert_close(det, ores[0][0], 1e-4, f'merged detections (rescale={rescale})')
        assert_close(det, torch.from_numpy(gold[f'det_rescale{int(rescale)}']), 1e-4, 'vs reference golden')
        # the boxes are exact copies of mapped-back inputs whose arithmetic is IEEE add / sub / div: bit equal
        assert torch.equal(det[:, :4], ores[0][0][:, :4])
