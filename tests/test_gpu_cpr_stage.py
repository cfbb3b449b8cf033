"""GPU parity of the CPR stage kernels (through the C ABI) against the oracle and the golden fixtures."""
import os

import numpy as np
import pytest
import torch

from oracle import cpr as ocpr, synth
from tests.helpers import assert_close, assert_mask_equal, flat_batch, oracle_cfg

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from pointtinybenchmark_b200 import ops
    return ops


def _extract(ops, inp, dev):
    d = inp['cfgd']
    fb, lens = flat_batch(inp, dev)
    off = ops.circle_offsets(d['radius'], d['stride']).to(dev)
    fmap = ops.to_nhwc(inp['cls_feat'].to(dev))
    feats, pts, valid = ops.bag_gather(fmap, fb['centers'], fb['bag_img'], off, d['stride'], fb['pad_hw'])
    return fb, lens, off, fmap, feats, pts, valid


@pytest.mark.parametrize('name,seed', [('lite', 1234), ('mid', 77)])
def test_gather_and_masks_vs_oracle_and_golden(ops, golden_dir, name, seed):
    dev = torch.device('cuda:0')
    inp = synth.cpr_inputs(name, seed)
    d = inp['cfgd']
    cfg = oracle_cfg(d)
    gold = np.load(os.path.join(golden_dir, f'cpr_{name}.npz'))
    fb, lens, off, fmap, feats, pts, valid = _extract(ops, inp, dev)
    gt_r = [p.reshape(len(l), -1, 2) for p, l in zip(ocpr.pseudo_bbox_to_center(inp['gt_bboxes']), inp['gt_labels'])]
    ex = ocpr.extract(inp['cls_feat'], gt_r, inp['gt_labels'], inp['img_metas'], cfg)
    # --- integer / bool outputs: bit exact
    assert_mask_equal(valid, ex['pos_valid'][:, 0, :, 0], 'pos_valid vs oracle')
    assert_mask_equal(valid, torch.from_numpy(gold['pos_valid'])[:, 0, :, 0], 'pos_valid vs golden')
    assert torch.equal(pts.cpu(), ex['pos_pts'][:, 0]), 'bag point coordinates must be bit-identical'
    assert torch.equal(pts.cpu(), torch.from_numpy(gold['pos_pts'])[:, 0])
    # --- gathered features: the kernel follows ATen's op order -> bit-exact (tests/test_gpu_bag_gather.py checks every path)
    ref = ex['pos_feats'][:, 0]
    nbad = int((feats.cpu() != ref).sum())
    assert torch.equal(feats.cpu(), ref), f'gathered features: {nbad} / {ref.numel()} values differ from the oracle'
    sub = feats.cpu().flatten()[::1009].numpy()
    assert np.abs(sub - gold['pos_feats_sub']).max() <= 1e-4 * max(1.0, np.abs(gold['pos_feats_sub']).max())
    # --- negative mask
    H, W = inp['cls_feat'].shape[2:]
    nm = ops.neg_mask(d['B'], H, W, d['stride'], fb['pad_hw'], fb['centers'], fb['labels'], fb['img_ptr'],
                      d['stride'] * d['radius'], d['num_classes'], True)
    assert_mask_equal(nm.reshape(-1, d['num_classes']), ex['neg_valid'], 'neg mask vs oracle')
    gneg = np.unpackbits(gold['neg_valid'])[:int(np.prod(gold['neg_valid_shape']))].reshape(gold['neg_valid_shape'])
    assert_mask_equal(nm.reshape(-1, d['num_classes']), torch.from_numpy(gneg.astype(bool)), 'neg mask vs golden')
    nm2 = ops.neg_mask(d['B'], H, W, d['stride'], fb['pad_hw'], fb['centers'], fb['labels'], fb['img_ptr'],
                       d['stride'] * d['radius'], d['num_classes'], False)
    ref2 = []
    for b in range(d['B']):
        g, gv = ocpr.anchor_points(H, W, *inp['img_metas'][b]['pad_shape'][:2], d['stride'])
        ref2.append(ocpr.out_circle_neg_mask(g.flatten(0, -2), gv.flatten(), gt_r[b], inp['gt_labels'][b], d['stride'],
                                             d['radius'], d['num_classes'], class_wise=False))
    assert_mask_equal(nm2.reshape(-1, d['num_classes']), torch.cat(ref2), 'class-agnostic neg mask')


@pytest.mark.parametrize('name,seed', [('lite', 1234), ('mid', 77)])
def test_linear_and_bag_logits(ops, golden_dir, name, seed):
    dev = torch.device('cuda:0')
    inp = synth.cpr_inputs(name, seed)
    d = inp['cfgd']
    gold = np.load(os.path.join(golden_dir, f'cpr_{name}.npz'))
    fb, lens, off, fmap, feats, pts, valid = _extract(ops, inp, dev)
    w = {k: v.to(dev) for k, v in inp['weights'].items()}
    G, K, C = feats.shape
    # reference dataflow: Linear on the gathered 256-d features
    lg = ops.linear_rows(feats.reshape(-1, C), w['cls_out.weight'], w['cls_out.bias']).reshape(G, K, -1)
    ref = torch.nn.functional.linear(feats.cpu(), inp['weights']['cls_out.weight'], inp['weights']['cls_out.bias'])
    e1 = assert_close(lg, ref, 1e-4, 'linear_rows vs F.linear')
    assert np.abs(lg.cpu().flatten()[::101].numpy() - gold['pos_cls_sub']).max() <= 1e-4 * np.abs(gold['pos_cls_sub']).max()
    # product dataflow: logit map first, then gather 80 channels (linearity of bilinear sampling)
    B, H, W, _ = fmap.shape
    wcat = torch.cat([w['cls_out.weight'], w['ins_out.weight']])
    bcat = torch.cat([w['cls_out.bias'], w['ins_out.bias']])
    lmap = ops.linear_rows(fmap.reshape(-1, C), wcat, bcat).reshape(B, H, W, -1)
    lg2, _, _ = ops.bag_gather(lmap, fb['centers'], fb['bag_img'], off, d['stride'], fb['pad_hw'], pts=False, valid=False)
    ncls = d['num_classes']
    e2 = assert_close(lg2[..., :ncls], ref, 1e-4, 'logit-map path vs reference dataflow')
    ref_ins = torch.nn.functional.linear(feats.cpu(), inp['weights']['ins_out.weight'], inp['weights']['ins_out.bias'])
    e3 = assert_close(lg2[..., ncls:], ref_ins, 1e-4, 'ins logits')
    print(f'[{name}] linear err {e1:.2e}; fused-order cls err {e2:.2e}; ins err {e3:.2e}')


@pytest.mark.parametrize('name,seed', [('lite', 1234), ('mid', 77)])
def test_refine_stage_and_fused(ops, golden_dir, name, seed):
    dev = torch.device('cuda:0')
    inp = synth.cpr_inputs(name, seed)
    d = inp['cfgd']
    cfg = oracle_cfg(d)
    gold = np.load(os.path.join(golden_dir, f'cpr_{name}.npz'))
    fb, lens, off, fmap, feats, pts, valid = _extract(ops, inp, dev)
    res, allo = ocpr.cpr_get_bboxes(inp['cls_feat'], inp['weights'], inp['gt_bboxes'], inp['gt_labels'], inp['gt_anns_id'],
                                    inp['img_metas'], cfg, return_all=True)
    ora = {k: torch.cat([r[k] for r in allo['refine']]) for k in allo['refine'][0]}
    groups = ops.label_groups(fb['bag_img'], fb['labels'], d['num_classes'])
    rc = ops._refine_cfg(cfg['merge_th'], cfg['gt_alpha'], cfg['refine_th'], True, True, False)
    # ---- stage kernel on the ORACLE's probabilities: every mask must be bit exact
    prob = allo['bag_prob'][:, 0].contiguous().to(dev)
    o_pts, o_sc, o_nr, o_ch, o_mv = ops.refine(prob, pts, valid, pts.shape[1], fb['labels'], fb['bag_img'], fb['img_hw'],
                                               groups, rc)
    assert_mask_equal(o_mv, ora['merge_valid'], 'merge_valid (stage)')
    assert_mask_equal(o_ch, ora['chosen'], 'chosen (stage)')
    assert_mask_equal(o_nr, ora['not_refine'], 'not_refine (stage)')
    assert_mask_equal(o_mv, torch.from_numpy(gold['merge_valid']), 'merge_valid vs golden')
    assert_mask_equal(o_nr, torch.from_numpy(gold['not_refine']), 'not_refine vs golden')
    assert_close(o_pts, ora['refine_pts'], 1e-4, 'refined points (stage)')
    assert_close(o_sc, ora['refine_scores'], 1e-4, 'refine scores (stage)')
    # filters one by one
    for flags, key in [((True, False), 'mask_nearest'), ((False, True), 'mask_classify')]:
        rcf = ops._refine_cfg(-1.0, 0.0, cfg['refine_th'], flags[0], flags[1], False)
        _, _, _, _, mv = ops.refine(prob, pts, torch.ones_like(valid), pts.shape[1], fb['labels'], fb['bag_img'],
                                    fb['img_hw'] * 0 + 100000, groups, rcf)
        nonneg = ((pts[..., 0] >= 0) & (pts[..., 1] >= 0)).cpu()      # the inside-image test cannot be switched off
        assert_mask_equal(mv, ora[key] & nonneg, key)
        assert_mask_equal(mv, torch.from_numpy(gold[key]) & nonneg, key + ' vs golden')
    # ---- fused kernel: logits computed on the GPU.  masks may differ from the oracle only where the oracle's
    # own float margin is below tolerance; the fixtures are built so that this set is empty.
    w = {k: v.to(dev) for k, v in inp['weights'].items()}
    B, H, W, C = fmap.shape
    lmap = ops.linear_rows(fmap.reshape(-1, C), w['cls_out.weight'], w['cls_out.bias']).reshape(B, H, W, -1)
    f_pts, f_sc, f_nr, f_ch = ops.refine_fused(lmap, d['num_classes'], fb['centers'], fb['labels'], fb['bag_img'], off,
                                               d['stride'], fb['pad_hw'], fb['img_hw'], groups, rc, want_chosen=True)
    nbad = int((f_ch.cpu() != ora['chosen']).sum())
    print(f'[{name}] fused refine: chosen-mask mismatches {nbad}/{f_ch.numel()}, not_refine mismatches '
          f'{int((f_nr.cpu() != ora["not_refine"]).sum())}')
    assert_mask_equal(f_nr, ora['not_refine'], 'not_refine (fused)')
    assert_mask_equal(f_ch, ora['chosen'], 'chosen (fused)')
    assert_close(f_pts, ora['refine_pts'], 1e-4, 'refined points (fused)')
    assert_close(f_sc, ora['refine_scores'], 1e-4, 'refine scores (fused)')
    det = torch.cat([r[0] for r in res])
    boxes = torch.cat([f_pts - 8, f_pts + 8, f_sc[:, None]], 1).cpu()
    assert_close(boxes, det[:, :5], 1e-4, 'pseudo boxes vs oracle get_bboxes')
    assert_close(boxes, torch.from_numpy(gold['det'])[:, :5], 1e-4, 'pseudo boxes vs golden')
