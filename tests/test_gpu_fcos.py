"""GPU: FCOSHead (pointtinybenchmark_b200/fcos_head.py, csrc/fcos.cu) against the reference's golden fixtures (oracle/make_golden_fcos.py):
forward, targets, losses and gradients, the training step through the towers, get_bboxes on both NMS routes, aug_test over tiles, and
every constructor refusal."""
import os

import numpy as np
import pytest
import torch

from oracle import fcos as ofc

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def gold(name):
    return np.load(os.path.join(GOLD, f'fcos_{name}.npz'))


def rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / max(1.0, float(b.abs().max()))) if b.numel() else 0.0


def make_head(name, **over):
    from pointtinybenchmark_b200.fcos_head import FCOSHead
    kw = dict(ofc.head_kwargs(name), **over)
    h = FCOSHead(**kw).cuda()
    h.load_state_dict({k: v.cuda() for k, v in ofc.case_inputs(name)['weights'].items()}, strict=True)
    return h


def maps_of(g, key, L=5):
    return tuple([torch.from_numpy(g[f'{key}_{n}{l}']).cuda() for l in range(L)] for n in ('cls', 'reg', 'ctr'))


def case_maps(name):
    g = gold(name)
    if f'eval_cls0' in g:
        return maps_of(g, 'train'), maps_of(g, 'eval')
    m = tuple([t.cuda() for t in ts] for ts in ofc.case_inputs(name)['maps'])
    return m, m


def cuda_gts(inp):
    return [b.cuda() for b in inp['gt_bboxes']], [l.cuda() for l in inp['gt_labels']]


@pytest.mark.parametrize('name', ['tinyperson', 'options'])
def test_forward_matches_reference(name):
    g, inp = gold(name), ofc.case_inputs(name)
    head = make_head(name).eval()
    with torch.no_grad():
        out = head([f.cuda() for f in inp['feats']])
    for n, ts in zip(('cls', 'reg', 'ctr'), out):
        for l, t in enumerate(ts):
            assert rel(t, g[f'eval_{n}{l}']) < 1e-4, (n, l)        # includes the 4 x 5 stride-128 map of a 640 x 512 tile
    assert head.last_tower_backend == 'wgmma-f16x2'


@pytest.mark.parametrize('name', ['tinyperson', 'coco80', 'options', 'no_pos'])
def test_targets_bit_exact(name):
    g, inp = gold(name), ofc.case_inputs(name)
    head = make_head(name)
    pts = head.get_points(inp['sizes'], torch.float32, 'cuda')
    labels, targets = head.get_targets(pts, *cuda_gts(inp))
    for l in range(5):
        assert torch.equal(labels[l].cpu(), torch.from_numpy(g[f'labels{l}'].astype(np.int64))), l
        assert torch.equal(targets[l].cpu(), torch.from_numpy(g[f'bbox_targets{l}'])), l


def _grad_check(t, g, key, tol):
    if key in g:
        assert rel(t, g[key]) < tol, key
    else:
        f = t.detach().flatten().double().cpu()
        assert rel(f[::7], g[key + '_sub']) < tol, key
        assert abs(float(f.sum()) - float(g[key + '_sum'])) <= tol * max(1.0, float(g[key + '_abssum'])), key


@pytest.mark.parametrize('name', ['tinyperson', 'coco80', 'options', 'no_pos'])
def test_loss_from_reference_maps_without_host_sync(name):
    g, inp = gold(name), ofc.case_inputs(name)
    head = make_head(name).train()
    train_maps, _ = case_maps(name)
    maps = tuple([t.clone().requires_grad_(True) for t in ts] for ts in train_maps)
    gts, gls = cuda_gts(inp)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        losses = head.loss(*maps, gts, gls, inp['img_metas'])
        sum(losses.values()).backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for k in ('loss_cls', 'loss_bbox', 'loss_centerness'):
        assert rel(losses[k].detach(), g[k]) < 1e-4, (k, float(losses[k]), float(g[k]))
    for n, ts in zip(('cls', 'reg', 'ctr'), maps):
        for l, t in enumerate(ts):
            key = f'grad_{n}{l}'
            if key in g or key + '_sub' in g:
                _grad_check(t.grad, g, key, 2e-4)
    if name == 'no_pos':
        assert float(losses['loss_bbox'].detach()) == 0.0 and float(losses['loss_centerness'].detach()) == 0.0
        assert not any(t.grad.any() for t in maps[1] + maps[2])


@pytest.mark.parametrize('name', ['tinyperson', 'options'])
def test_training_step_parameter_gradients(name):
    g, inp = gold(name), ofc.case_inputs(name)
    head = make_head(name).train()
    losses = head.loss(*head([f.cuda() for f in inp['feats']]), *cuda_gts(inp), inp['img_metas'])
    sum(losses.values()).backward()
    assert head.last_tower_backend == 'wgmma-f16x2-train'
    for k in ('loss_cls', 'loss_bbox', 'loss_centerness'):
        assert rel(losses[k].detach(), g[k]) < 1e-4, k
    errs = {}
    for k, p in head.named_parameters():
        key = f'pgrad/{k}'
        if p.dim() == 4:
            # conv weight gradients by norm, as tests/test_gpu_p2p_multilevel.py compares the tower's: pre-activations within rounding of
            # zero pass the GroupNorm + ReLU layers gated differently, and the output convs' weight gradients sum the fp16-pair towers'
            # features over every cell, so single elements move far more than the sums do
            f = p.grad.flatten()[::97] if key + '_sub' in g else p.grad.flatten()
            ref_ = torch.from_numpy(g[key + '_sub'] if key + '_sub' in g else g[key]).double().flatten()
            errs[k] = (float((f.double().cpu() - ref_).norm() / ref_.norm()),
                       3e-2 if k.startswith('reg_convs') else 5e-3 if k.startswith('cls_convs') else 2e-3)
        else:
            errs[k] = (rel(p.grad, g[key]), 2e-4)
    assert all(e <= tol for e, tol in errs.values()), {k: v for k, v in errs.items() if v[0] > v[1]}


def _same_up_to_equal_keys(got, ref, keys):
    """row sets equal, and orders equal except inside groups of exactly equal fp32 keys"""
    assert len(got) == len(ref)
    assert torch.equal(keys[got], keys[ref])
    for v in torch.unique(keys[ref]):
        assert set(got[keys[got] == v].tolist()) == set(ref[keys[ref] == v].tolist())


@pytest.mark.parametrize('name', ['tinyperson', 'coco80', 'options', 'no_pos'])
def test_get_bboxes_from_reference_maps(name):
    g, inp = gold(name), ofc.case_inputs(name)
    c = ofc.CASES[name]
    head = make_head(name).eval()
    _, emaps = case_maps(name)
    rescale = c.get('rescale', False)
    idx, boxes, scores, ctr = head._decode(*emaps, inp['img_metas'], head.test_cfg, rescale)
    # top-k rows per level against the reference's keys
    B, C, off = len(inp['img_metas']), c['head']['num_classes'], 0
    for l, (h, w) in enumerate(inp['sizes']):
        n = ofc.fcos_rows(h * w, c['test']['nms_pre'])
        if f'topk{l}' in g:
            key = (emaps[0][l].cpu().sigmoid() * emaps[2][l].cpu().sigmoid()).permute(0, 2, 3, 1).reshape(B, -1, C).max(-1)[0].cpu()
            for b in range(B):
                _same_up_to_equal_keys(idx[b, off:off + n].long().cpu(), torch.from_numpy(g[f'topk{l}'][b]).long(), key[b])
        off += n
    res = head.get_bboxes(*emaps, inp['img_metas'], rescale=rescale)
    for b, (d, lab) in enumerate(res):
        rd, rl = torch.from_numpy(g[f'dets{b}']), torch.from_numpy(g[f'det_labels{b}'].astype(np.int64))
        assert d.shape == rd.shape, (b, d.shape, rd.shape)
        assert torch.equal(lab.cpu(), rl)
        assert rel(d, rd) < 1e-4


def test_get_bboxes_batched_nms_route():
    """nms_pre=-1 keeps all 6 820 rows of a 640 x 512 tile: more than the multiclass kernels' 4096, so ptb_batched_nms runs"""
    inp = ofc.case_inputs('tinyperson')
    _, emaps = case_maps('tinyperson')
    test_cfg = dict(ofc.TINY_TEST, nms_pre=-1)
    head = make_head('tinyperson', test_cfg=test_cfg).eval()
    res = head.get_bboxes(*emaps, inp['img_metas'])
    ref, _ = ofc.get_bboxes(*[[t.cpu() for t in ts] for ts in emaps], inp['img_metas'], ofc.TINY, test_cfg)
    for (d, l), (rd, rl) in zip(res, ref):
        assert d.shape == rd.shape
        assert torch.equal(l.cpu(), rl)
        assert rel(d, rd) < 1e-4


@pytest.mark.parametrize('name', ['tiles', 'flip_scale'])
@pytest.mark.parametrize('rescale', [False, True])
def test_aug_test_from_reference_maps(name, rescale):
    g = gold(name)
    augs = ofc.tile_case(name)
    assert g['seeds'].tolist() == [a['seed'] for a in augs]
    maps = [tuple([t.cuda() for t in ts] for ts in ofc.aug_maps(a)) for a in augs]
    head = make_head('tinyperson').eval()
    by_shape = {}
    for m in maps:
        by_shape.setdefault(tuple(tuple(t.shape) for t in m[0]), []).append(m)
    # the head batches augs of one shape: its forward gets their features concatenated and returns their maps concatenated
    head.forward = lambda x: tuple([torch.cat([m[k][l] for m in by_shape[tuple((1,) + tuple(t.shape[1:]) for t in x)][:x[0].shape[0]]])
                                    for l in range(5)] for k in range(3))
    feats = [[torch.zeros(1, 1, h, w, device='cuda') for h, w in a['sizes']] for a in augs]
    d, lab = head.aug_test([f for f in feats], [[a['meta']] for a in augs], rescale=rescale)[0]
    rd, rl = torch.from_numpy(g[f'dets_rescale{int(rescale)}']), torch.from_numpy(g[f'labels_rescale{int(rescale)}'].astype(np.int64))
    assert d.shape == rd.shape
    assert torch.equal(lab.cpu(), rl)
    assert rel(d, rd) < 1e-4


@pytest.mark.parametrize('over, msg', [
    (dict(norm_cfg=None), 'norm_cfg=None'),
    (dict(dcn_on_last_conv=True), 'dcn_on_last_conv'),
    (dict(conv_bias=True), 'conv_bias=True'),
    (dict(feat_channels=128), 'feat_channels=128'),
    (dict(num_classes=512), 'at most 511 classes'),
    (dict(loss_bbox=dict(type='DIoULoss')), 'IoULoss and GIoULoss'),
    (dict(loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=True)), 'FocalLoss'),
    (dict(loss_centerness=dict(type='MSELoss')), 'CrossEntropyLoss'),
])
def test_refusals(over, msg):
    from pointtinybenchmark_b200.fcos_head import FCOSHead
    with pytest.raises(NotImplementedError, match=msg):
        FCOSHead(**dict(ofc.head_kwargs('tinyperson'), **over))
