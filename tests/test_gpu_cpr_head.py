"""GPU parity of the CPRHead plugin (loss + gradients, get_bboxes) against the oracle and the golden fixtures."""
import os

import numpy as np
import pytest
import torch

from oracle import cpr as ocpr, synth
from tests.helpers import assert_close, assert_mask_equal, oracle_cfg

pytestmark = pytest.mark.gpu


def head_cfg(d):
    r = d['radius']
    return dict(
        type='CPRHead', norm_cfg=dict(type='GN', num_groups=32, requires_grad=True),
        num_classes=d['num_classes'], in_channels=d['C'], feat_channels=d['C'], stacked_convs=4, num_cls_fcs=0,
        strides=[d['stride']],
        loss_mil=dict(type='MILLoss', binary_ins=False, loss_weight=0.25), loss_type=0,
        loss_cfg=dict(with_neg=True, neg_loss_weight=0.75, refine_bag_policy='only_refine_bag', random_remove_rate=0.4,
                      with_gt_loss=True, gt_loss_weight=0.125, with_mil_loss=True),
        normal_cfg=dict(prob_cls_type='sigmoid', out_bg_cls=False),
        train_pts_extractor=dict(pos_generator=dict(type='CirclePtFeatGenerator', radius=r),
                                 neg_generator=dict(type='OutCirclePtFeatGenerator', radius=r, class_wise=True)),
        refine_pts_extractor=dict(pos_generator=dict(type='CirclePtFeatGenerator', radius=r),
                                  neg_generator=dict(type='OutCirclePtFeatGenerator', radius=r, keep_wh=True, class_wise=True)),
        point_refiner=dict(merge_th=0.1, refine_th=0.1, classify_filter=True, nearest_filter=True),
        train_cfg=None, test_cfg=dict(nms_pre=1000, score_thr=0.05, nms=dict(type='nms', iou_threshold=0.5), max_per_img=100))


@pytest.fixture(scope='module')
def build():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from pointtinybenchmark_b200 import cpr_head  # noqa: F401  (registers the head)
    from pointtinybenchmark_b200.registry import build_head

    def _b(inp):
        head = build_head(head_cfg(inp['cfgd'])).cuda()
        sd = head.state_dict()
        sd.update({k: v for k, v in inp['weights'].items()})
        head.load_state_dict(sd, strict=True)
        return head
    return _b


def _to_dev(inp, dev):
    return ([b.to(dev) for b in inp['gt_bboxes']], [l.to(dev) for l in inp['gt_labels']], [a.to(dev) for a in inp['gt_anns_id']])


@pytest.mark.parametrize('name,seed', [('lite', 1234), ('mid', 77)])
def test_loss_and_grads(build, golden_dir, name, seed):
    dev = torch.device('cuda:0')
    inp = synth.cpr_inputs(name, seed)
    cfg = oracle_cfg(inp['cfgd'])
    gold = np.load(os.path.join(golden_dir, f'cpr_{name}.npz'))
    head = build(inp)
    gtb, gtl, _ = _to_dev(inp, dev)
    feat = inp['cls_feat'].to(dev).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    losses = head.loss([feat], [feat], gtb, gtl, inp['img_metas'])
    total = sum(v for k, v in losses.items() if 'loss' in k)
    total.backward()
    # oracle with autograd on the CPU
    fo = inp['cls_feat'].clone().requires_grad_(True)
    wo = {k: v.clone().requires_grad_(True) for k, v in inp['weights'].items()}
    ol = ocpr.cpr_loss(fo, wo, inp['gt_bboxes'], inp['gt_labels'], inp['img_metas'], cfg)
    sum(v for k, v in ol.items() if 'loss' in k).backward()
    for k in ('gt_loss', 'pos_loss', 'neg_loss', 'bag_acc'):
        e = assert_close(losses[k].reshape(-1), ol[k].detach().reshape(-1), 1e-4, k)
        assert_close(losses[k].reshape(-1), torch.from_numpy(gold['loss_' + k]), 1e-4, k + ' vs golden')
        print(f'[{name}] {k}: {float(losses[k].reshape(-1)[0]):.6f} (oracle {float(ol[k].reshape(-1)[0]):.6f}, err {e:.1e})')
    e = assert_close(feat.grad, fo.grad, 2e-4, 'd loss / d feature map')
    sub = feat.grad.detach().cpu().contiguous().flatten()[::211].numpy()
    assert np.abs(sub - gold['grad_feat_sub']).max() <= 2e-4 * np.abs(gold['grad_feat_sub']).max()
    e2 = assert_close(head.cls_out.weight.grad, wo['cls_out.weight'].grad, 2e-4, 'd/d cls_out.weight')
    e3 = assert_close(head.ins_out.weight.grad, wo['ins_out.weight'].grad, 2e-4, 'd/d ins_out.weight')
    assert_close(head.cls_out.bias.grad, wo['cls_out.bias'].grad, 2e-4, 'd/d cls_out.bias')
    # softmax over the bag is shift invariant: the ins bias gradient is analytically zero (fp noise on both sides)
    wscale = float(wo['ins_out.weight'].grad.abs().max())
    assert float((head.ins_out.bias.grad.cpu() - wo['ins_out.bias'].grad).abs().max()) <= 1e-5 * wscale
    assert_close(head.cls_out.weight.grad, torch.from_numpy(gold['grad_cls_w']), 2e-4, 'dW cls vs golden')
    assert_close(head.ins_out.weight.grad, torch.from_numpy(gold['grad_ins_w']), 2e-4, 'dW ins vs golden')
    print(f'[{name}] grad errs: feat {e:.1e}, Wcls {e2:.1e}, Wins {e3:.1e}')


@pytest.mark.parametrize('name,seed', [('lite', 1234), ('mid', 77)])
def test_get_bboxes(build, golden_dir, name, seed):
    dev = torch.device('cuda:0')
    inp = synth.cpr_inputs(name, seed)
    cfg = oracle_cfg(inp['cfgd'])
    gold = np.load(os.path.join(golden_dir, f'cpr_{name}.npz'))
    head = build(inp).eval()
    gtb, gtl, aid = _to_dev(inp, dev)
    feat = inp['cls_feat'].to(dev)
    res, nr = head.get_bboxes([feat], [feat], inp['img_metas'], gt_bboxes=gtb, gt_labels=gtl, gt_anns_id=aid,
                              cascade_out_fmt=True)
    ora = ocpr.cpr_get_bboxes(inp['cls_feat'], inp['weights'], inp['gt_bboxes'], inp['gt_labels'], inp['gt_anns_id'],
                              inp['img_metas'], cfg)
    assert len(res) == len(ora)
    for b in range(len(res)):
        assert res[b][0].shape == ora[b][0].shape
        assert_close(res[b][0][:, :5], ora[b][0][:, :5], 1e-4, f'det[{b}]')
        assert torch.equal(res[b][0][:, 5].cpu(), ora[b][0][:, 5]), 'ann ids'
        assert torch.equal(res[b][1].cpu(), ora[b][1])
    assert_mask_equal(torch.cat(nr), torch.from_numpy(gold['not_refine']), 'not_refine vs golden')
    assert_close(torch.cat([r[0] for r in res]), torch.from_numpy(gold['det']), 1e-4, 'det vs golden')
    # second pass of a cascade: carried not_refine must stick (cpr_head.py:837)
    res2, nr2 = head.get_bboxes([feat], [feat], inp['img_metas'], gt_bboxes=gtb, gt_labels=gtl, gt_anns_id=aid,
                                not_refine=[torch.ones_like(x) for x in nr], cascade_out_fmt=True)
    assert bool(torch.cat(nr2).all())
    pts = torch.cat([(b[:, :2] + b[:, 2:]) / 2 for b in gtb])
    got = torch.cat([r[0] for r in res2])
    assert torch.equal((got[:, :2] + got[:, 2:4]) / 2, pts)


def test_tower_forward_matches_oracle(build, golden_dir):
    dev = torch.device('cuda:0')
    inp = synth.cpr_inputs('lite', 99, with_towers=True)
    cfg = oracle_cfg(inp['cfgd'])
    head = build(inp).eval()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    with torch.no_grad():
        out = head([inp['cls_feat'].to(dev)])[0][0]
        ref = ocpr.tower_forward(inp['cls_feat'], inp['weights'], cfg)
    assert_close(out, ref, 1e-4, 'conv towers (cuDNN fp32) vs oracle')
    gold = np.load(os.path.join(golden_dir, 'cpr_lite_tower.npz'))
    sub = out.cpu().contiguous().flatten()[::97].numpy()
    assert np.abs(sub - gold['tower_sub']).max() <= 1e-4 * np.abs(gold['tower_sub']).max()


def test_one_class_head_and_empty_image(build):
    """ragged / degenerate inputs: 1 class (TinyPerson-style), an image with a single GT, points on the border."""
    dev = torch.device('cuda:0')
    inp = synth.cpr_inputs('mid', 5, num_classes=1, n=3)
    inp['gt_bboxes'][1] = inp['gt_bboxes'][1][:1]
    inp['gt_labels'][1] = inp['gt_labels'][1][:1]
    inp['gt_anns_id'][1] = inp['gt_anns_id'][1][:1]
    inp['gt_bboxes'][0][0] = torch.tensor([-8., -8., 8., 8.])      # centre exactly at (0,0)
    cfg = oracle_cfg(inp['cfgd'])
    head = build(inp)
    gtb, gtl, aid = _to_dev(inp, dev)
    feat = inp['cls_feat'].to(dev).requires_grad_(True)
    losses = head.loss([feat], [feat], gtb, gtl, inp['img_metas'])
    sum(v for k, v in losses.items() if 'loss' in k).backward()
    fo = inp['cls_feat'].clone().requires_grad_(True)
    ol = ocpr.cpr_loss(fo, inp['weights'], inp['gt_bboxes'], inp['gt_labels'], inp['img_metas'], cfg)
    sum(v for k, v in ol.items() if 'loss' in k).backward()
    for k in ('gt_loss', 'pos_loss', 'neg_loss'):
        assert_close(losses[k].reshape(-1), ol[k].detach().reshape(-1), 1e-4, k)
    assert_close(feat.grad, fo.grad, 2e-4, 'grad (1 class)')
    res = head.get_bboxes([feat.detach()], [feat.detach()], inp['img_metas'], gt_bboxes=gtb, gt_labels=gtl, gt_anns_id=aid)
    ora = ocpr.cpr_get_bboxes(inp['cls_feat'], inp['weights'], inp['gt_bboxes'], inp['gt_labels'], inp['gt_anns_id'],
                              inp['img_metas'], cfg)
    for b in range(2):
        assert_close(res[b][0][:, :5], ora[b][0][:, :5], 1e-4, f'det[{b}] (1 class)')


@pytest.mark.parametrize('rescale', [False, True])
def test_get_bboxes_out_geo(build, rescale):
    """other_info.out_geo (cpr_head.py:855-866, 1262-1273): rows grow by [refined point, chosen bag points ...] padded with -1 to
    the longest list of the image; the chosen SET is a bit-exact target, the coordinates are exact copies of bag points."""
    dev = torch.device('cuda:0')
    inp = synth.cpr_inputs('mid', 77)
    cfg = oracle_cfg(inp['cfgd'])
    from pointtinybenchmark_b200.registry import build_head
    hc = head_cfg(inp['cfgd'])
    hc['other_info'] = dict(out_geo=True)
    head = build_head(hc).cuda().eval()
    sd = head.state_dict()
    sd.update(inp['weights'])
    head.load_state_dict(sd, strict=True)
    gtb, gtl, aid = _to_dev(inp, dev)
    metas = [dict(m, scale_factor=[1.5, 1.25, 1.5, 1.25]) for m in inp['img_metas']]
    feat = inp['cls_feat'].to(dev)
    res = head.get_bboxes([feat], [feat], metas, rescale=rescale, gt_bboxes=gtb, gt_labels=gtl, gt_anns_id=aid)
    ora = ocpr.cpr_get_bboxes(inp['cls_feat'], inp['weights'], inp['gt_bboxes'], inp['gt_labels'], inp['gt_anns_id'], metas, cfg,
                              rescale=rescale, out_geo=True)
    for b in range(len(res)):
        a, o = res[b][0].cpu(), ora[b][0]
        assert a.shape == o.shape and a.shape[1] > 8
        assert torch.equal(a[:, 8:] < 0, o[:, 8:] < 0), 'geo padding pattern (= number of chosen points per GT)'
        assert torch.equal(a[:, 8:], o[:, 8:]), 'chosen bag points are exact copies'
        assert_close(a[:, :8], o[:, :8], 1e-4, 'box, score, ann id, refined point')


def test_config5_shape_two_pass_refine(build):
    """BASELINE.json configs[4] per-GPU shard shape: 2000 points per image (578 k bag samples / image), 'multi-scale refine' emulated as
    two sequential get_bboxes passes feeding the refined points back with `not_refine` carried (SURVEY.md §8d), checked through
    size-independent properties (determinism, carried not_refine, fixed points); oracle parity at this shape: test_gpu_full_shape.py."""
    dev = torch.device('cuda:0')
    inp = synth.cpr_inputs('cpr2000', 31, B=2)
    head = build(inp).eval()
    gtb, gtl, aid = _to_dev(inp, dev)
    feat = inp['cls_feat'].to(dev)
    metas = inp['img_metas']
    res1, nr1 = head.get_bboxes([feat], [feat], metas, gt_bboxes=gtb, gt_labels=gtl, gt_anns_id=aid, cascade_out_fmt=True)
    res1b, nr1b = head.get_bboxes([feat], [feat], metas, gt_bboxes=gtb, gt_labels=gtl, gt_anns_id=aid, cascade_out_fmt=True)
    for a, b in zip(res1, res1b):
        assert torch.equal(a[0], b[0]), 'deterministic'
    assert all(r[0].shape == (2000, 6) for r in res1)
    frac = float(torch.cat(nr1).float().mean())
    assert 0.02 < frac < 0.7, frac
    # (the oracle comparison at this shape lives in tests/test_gpu_full_shape.py::test_config5_shape_margin_harness: float64 decision
    #  margins, bit-equality wherever the margin exceeds the bound — no 'a few rows may differ' allowance)
    # second pass on the refined points
    gtb2 = [r[0][:, :4].contiguous() for r in res1]
    res2, nr2 = head.get_bboxes([feat], [feat], metas, gt_bboxes=gtb2, gt_labels=gtl, gt_anns_id=aid, not_refine=nr1,
                                cascade_out_fmt=True)
    for b in range(len(res1)):
        assert bool((nr2[b] | ~nr1[b]).all()), 'not_refine is carried (cpr_head.py:837)'
        keep = nr1[b]
        assert torch.equal(res2[b][0][keep, :4], res1[b][0][keep, :4]), 'points that were not refined stay where they are'
        c2 = (res2[b][0][:, :2] + res2[b][0][:, 2:4]) / 2
        assert bool((c2[:, 0] >= -64).all() and (c2[:, 0] <= 1344 + 64).all() and (c2[:, 1] >= -64).all() and (c2[:, 1] <= 800 + 64).all())
    moved = float(((res2[0][0][:, :2] - res1[0][0][:, :2]).abs().max(dim=1)[0] > 1e-3).float().mean())
    print(f'[config 5 shape] not_refine pass 1 {frac:.3f}, pass 2 {float(torch.cat(nr2).float().mean()):.3f}; points moved again in pass 2: {moved:.3f}')


def test_training_gradients_are_deterministic(build):
    """VERDICT r1 #8: the loss path's scatter (grid_sample backward) used fp32 atomics.  In the deterministic mode
    (torch.use_deterministic_algorithms(True) or PTB_LOSS_BWD=tiles) the map gradient comes from the tile-owner kernel (every sum formed by
    one thread in a fixed order) and the weight gradients from fixed-order tensor-core reductions: feat.grad and every parameter gradient
    of the head must be BIT-IDENTICAL across runs (heavily overlapping bags: 300 points on a 24x36 map).  The default mode (fused
    scatter, fp32 vector atomics) and round 1's staged chain must agree with it within the gradient tolerance."""
    dev = torch.device('cuda:0')
    inp = synth.cpr_inputs('mid', 123, n=150)
    head = build(inp)
    gtb, gtl, _ = _to_dev(inp, dev)

    def run(mode):
        if mode is None:
            os.environ.pop('PTB_LOSS_BWD', None)
        else:
            os.environ['PTB_LOSS_BWD'] = mode
        try:
            head.zero_grad(set_to_none=True)
            feat = inp['cls_feat'].to(dev).contiguous(memory_format=torch.channels_last).requires_grad_(True)
            losses = head.loss([feat], [feat], gtb, gtl, inp['img_metas'])
            sum(v for k, v in losses.items() if 'loss' in k).backward()
            return [feat.grad.clone()] + [p.grad.clone() for p in (head.cls_out.weight, head.cls_out.bias, head.ins_out.weight, head.ins_out.bias)]
        finally:
            os.environ.pop('PTB_LOSS_BWD', None)
    grads = [run('tiles') for _ in range(3)]
    for other in grads[1:]:
        for a, b in zip(grads[0], other):
            assert torch.equal(a, b), 'gradients differ between two runs on identical inputs (deterministic mode)'
    torch.use_deterministic_algorithms(True)
    try:
        again = run(None)
    finally:
        torch.use_deterministic_algorithms(False)
    assert all(torch.equal(a, b) for a, b in zip(grads[0], again)), 'torch.use_deterministic_algorithms(True) must select the tile kernel'
    for mode in (None, 'staged'):
        other = run(mode)
        assert_close(other[0], grads[0][0], 2e-4, f'mode {mode}: d loss / d feature map')
        assert_close(other[1], grads[0][1], 2e-4, f'mode {mode}: dW cls')
        assert_close(other[3], grads[0][3], 2e-4, f'mode {mode}: dW ins')


@pytest.mark.parametrize('deterministic', [False, True])
@pytest.mark.parametrize('N', [1, 10, 33, 100])
def test_loss_and_grads_class_counts(build, N, deterministic):
    """CPRHead.loss + backward against the oracle at class counts other than 80, in the default mode and under
    torch.use_deterministic_algorithms(True).  Deterministic mode pads the logit rows to NP = ceil16(N) (LD = 32, 32, 96 here, so the
    1-tap wgmma GEMMs run with 32- and 96-column operands) and must give bit-identical gradients on two runs; at N = 100 it has no tile
    kernel and must raise, or warn and run the atomic path in warn-only mode."""
    dev = torch.device('cuda:0')
    inp = synth.cpr_inputs('lite', 500 + N, num_classes=N)
    cfg = oracle_cfg(inp['cfgd'])
    head = build(inp)
    gtb, gtl, _ = _to_dev(inp, dev)

    def run():
        head.zero_grad(set_to_none=True)
        feat = inp['cls_feat'].to(dev).contiguous(memory_format=torch.channels_last).requires_grad_(True)
        losses = head.loss([feat], [feat], gtb, gtl, inp['img_metas'])
        sum(v for k, v in losses.items() if 'loss' in k).backward()
        return losses, [feat.grad.clone()] + [p.grad.clone() for p in (head.cls_out.weight, head.cls_out.bias, head.ins_out.weight)]

    os.environ.pop('PTB_LOSS_BWD', None)
    torch.use_deterministic_algorithms(deterministic)
    try:
        if deterministic and N > 80:
            with pytest.raises(RuntimeError, match='no deterministic implementation'):
                run()
            torch.use_deterministic_algorithms(True, warn_only=True)
            with pytest.warns(UserWarning, match='no deterministic implementation'):
                losses, grads = run()
        else:
            losses, grads = run()
            if deterministic:
                _, again = run()
                assert all(torch.equal(a, b) for a, b in zip(grads, again)), f'N={N}: deterministic mode gave different gradient bits'
    finally:
        torch.use_deterministic_algorithms(False)
    fo = inp['cls_feat'].clone().requires_grad_(True)
    wo = {k: v.clone().requires_grad_(True) for k, v in inp['weights'].items()}
    ol = ocpr.cpr_loss(fo, wo, inp['gt_bboxes'], inp['gt_labels'], inp['img_metas'], cfg)
    sum(v for k, v in ol.items() if 'loss' in k).backward()
    errs = {k: assert_close(losses[k].reshape(-1), ol[k].detach().reshape(-1), 1e-4, f'N={N} {k}')
            for k in ('gt_loss', 'pos_loss', 'neg_loss', 'bag_acc')}
    errs['feat'] = assert_close(grads[0], fo.grad, 2e-4, f'N={N} d loss / d feature map')
    errs['Wcls'] = assert_close(grads[1], wo['cls_out.weight'].grad, 2e-4, f'N={N} dW cls')
    errs['bcls'] = assert_close(grads[2], wo['cls_out.bias'].grad, 2e-4, f'N={N} db cls')
    errs['Wins'] = assert_close(grads[3], wo['ins_out.weight'].grad, 2e-4, f'N={N} dW ins')
    print(f'[class counts] N={N} deterministic={deterministic}: ' + ', '.join(f'{k} {v:.1e}' for k, v in errs.items()))


def test_deterministic_mode_refuses_atomics(build):
    """an explicit PTB_LOSS_BWD=tiles that the tile kernel cannot serve raises even in warn-only mode, and PTB_LOSS_BWD=scatter under
    torch.use_deterministic_algorithms(True) raises: neither may run fp32 atomics silently."""
    dev = torch.device('cuda:0')
    inp = synth.cpr_inputs('lite', 9, num_classes=100)
    head = build(inp)
    gtb, gtl, _ = _to_dev(inp, dev)

    def run():
        feat = inp['cls_feat'].to(dev).requires_grad_(True)
        losses = head.loss([feat], [feat], gtb, gtl, inp['img_metas'])
        sum(v for k, v in losses.items() if 'loss' in k).backward()

    try:
        os.environ['PTB_LOSS_BWD'] = 'tiles'
        torch.use_deterministic_algorithms(True, warn_only=True)
        with pytest.raises(RuntimeError, match='num_classes=100'):
            run()
        torch.use_deterministic_algorithms(False)
        with pytest.raises(RuntimeError, match='num_classes=100'):
            run()
        os.environ['PTB_LOSS_BWD'] = 'scatter'
        torch.use_deterministic_algorithms(True)
        with pytest.raises(RuntimeError, match='PTB_LOSS_BWD=scatter'):
            run()
    finally:
        os.environ.pop('PTB_LOSS_BWD', None)
        torch.use_deterministic_algorithms(False)


def test_offsets_reach_follows_the_table(build):
    """the reach of an offset table belongs to the tensor, not to its address: a freed stride-4 table whose memory is handed to a
    stride-8 table of the same size must not lend it its (smaller) reach."""
    from pointtinybenchmark_b200 import ops
    from pointtinybenchmark_b200.cpr_head import _CircleBags
    dev = torch.device('cuda:0')
    a = ops.circle_offsets(3, 4).to(dev)
    ra = _CircleBags(a, 4.0).reach
    ptr = a.data_ptr()
    del a
    b = ops.circle_offsets(3, 8).to(dev)
    reused = b.data_ptr() == ptr
    assert ra == 12.0
    assert ops.offsets_reach(b) == 24.0 and _CircleBags(b, 8.0).reach == 24.0
    if not reused:
        pytest.skip('the caching allocator did not hand the freed table\'s address to the new one: the stale-reach case did not arise')


@pytest.mark.parametrize('variant', ['softmax', 'normed_sigmoid', 'fcs_binary'])
def test_head_variants_loss_grads_and_refine(golden_dir, variant):
    """the variants the reference class accepts beyond the shipped configs (cpr_head.py:1000-1008, 1055-1059, 1080-1099, 1108-1114;
    multi_instance_learning_loss.py:179-186): prob_cls_type softmax / normed_sigmoid (p = 2), num_cls_fcs = 2 + binary_ins, gt_weights.
    Generic path of the head (CUDA gather + torch elementwise) vs the oracle and the reference-pinned golden vectors."""
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from oracle.make_golden import CPR_VARIANTS, variant_weights
    from pointtinybenchmark_b200 import cpr_head  # noqa: F401
    from pointtinybenchmark_b200.registry import build_head
    dev = torch.device('cuda:0')
    inp = synth.cpr_inputs('lite', 4242)
    d = inp['cfgd']
    gold = np.load(os.path.join(golden_dir, f'cpr_lite_{variant}.npz'))
    hc = head_cfg(d)
    hc.update(CPR_VARIANTS[variant][0])
    head = build_head(hc).cuda()
    w = variant_weights(inp, variant, 4242)
    sd = head.state_dict()
    sd.update(w)
    head.load_state_dict(sd, strict=True)
    cfg = ocpr.default_cfg(num_classes=d['num_classes'], in_channels=d['C'], feat_channels=d['C'], stride=d['stride'], pos_radius=d['radius'],
                           neg_radius=d['radius'], **CPR_VARIANTS[variant][1])
    g = torch.Generator().manual_seed(4242 + 5)
    gtw = [torch.rand(len(l), generator=g) * 0.5 + 0.5 for l in inp['gt_labels']]
    gtw[0][0] = 0.0
    gtb, gtl, aid = _to_dev(inp, dev)
    feat = inp['cls_feat'].to(dev).requires_grad_(True)
    losses = head.loss([feat], [feat], gtb, gtl, inp['img_metas'], gt_weights=[t.to(dev) for t in gtw])
    sum(v for k, v in losses.items() if 'loss' in k).backward()
    fo = inp['cls_feat'].clone().requires_grad_(True)
    wo = {k: v.clone().requires_grad_(True) for k, v in w.items()}
    ol = ocpr.cpr_loss(fo, wo, inp['gt_bboxes'], inp['gt_labels'], inp['img_metas'], cfg, gt_weights=gtw)
    sum(v for k, v in ol.items() if 'loss' in k).backward()
    for k in ('gt_loss', 'pos_loss', 'neg_loss', 'bag_acc'):
        assert_close(losses[k].reshape(-1), ol[k].detach().reshape(-1), 1e-4, f'{variant} {k}')
        assert_close(losses[k].reshape(-1), torch.from_numpy(gold['loss_' + k]), 1e-4, f'{variant} {k} vs golden')
    assert_close(feat.grad, fo.grad, 2e-4, f'{variant} d loss / d feature map')
    assert_close(head.cls_out.weight.grad, wo['cls_out.weight'].grad, 2e-4, f'{variant} dW cls')
    assert_close(head.cls_out.weight.grad, torch.from_numpy(gold['grad_cls_w']), 2e-4, f'{variant} dW cls vs golden')
    head.eval()
    res, nr = head.get_bboxes([feat.detach()], [feat.detach()], inp['img_metas'], gt_bboxes=gtb, gt_labels=gtl, gt_anns_id=aid,
                              cascade_out_fmt=True)
    assert_mask_equal(torch.cat(nr), torch.from_numpy(gold['not_refine']), f'{variant} not_refine vs golden')
    assert_close(torch.cat([r[0] for r in res]), torch.from_numpy(gold['det']), 1e-4, f'{variant} det vs golden')
    # the inference entry point takes the same (generic) route for a variant head
    out = head.simple_test((torch.randn(1, 256, 32, 32, device=dev),), inp['img_metas'], gt_bboxes=gtb, gt_labels=gtl, gt_anns_id=aid)
    assert out[0][0].shape == (32, 6)
