"""GPU: P2PHead trained with GHMC, GHMR, L1Loss and BalancedL1Loss against the REAL reference's vectors
(tests/golden/p2p_loss_types_*.npz).  On the reference's own output maps: losses and map gradients within 1e-4, per-image bin counts
equal, acc_sum bit-identical after every step.  The full training step from the feature maps: losses and output-conv gradients within
1e-4 and the towers' gradients by norm where no GHMC decision lies near a bin edge.  Then the step repeating bit for bit under
torch.use_deterministic_algorithms(True), GHMC at 1203 classes (the wide cls_out path) and an fp16 feature map, each against the
oracle on the head's own logits."""
import os

import numpy as np
import pytest
import torch

from oracle import p2p_loss_types as olt, p2p_multilevel as oml
from oracle.make_golden_p2p_loss_types import GRAD_STEP, head_kwargs
from tests.test_gpu_p2p_defaults import TRAIN_CFG

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from pointtinybenchmark_b200 import ops
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return ops


def _close(a, ref_, tol, what):
    a, ref_ = np.asarray(a, np.float64), np.asarray(ref_, np.float64)
    assert a.shape == ref_.shape, (what, a.shape, ref_.shape)
    d = np.abs(a - ref_).max() if a.size else 0.0
    assert d <= tol * max(1.0, np.abs(ref_).max()), f'{what}: max |diff| {d:.3e}'


def build(cfg, weights):
    from pointtinybenchmark_b200.p2p_head import P2PHead
    head = P2PHead(**head_kwargs(cfg), train_cfg=TRAIN_CFG)
    head.load_state_dict(dict(weights, **olt.make_state(cfg)), strict=True)
    return head.cuda().train()


def _loss_args(inp):
    return [b.cuda() for b in inp['gt_bboxes']], [l.cuda() for l in inp['gt_labels']], inp['img_metas']


def _stack(v):
    return torch.stack([x.detach().reshape(()) for x in v]).cpu().numpy()


@pytest.mark.parametrize('name', sorted(olt.CASES))
def test_loss_on_reference_maps(ops, name):
    """head.loss on the oracle's output maps, which oracle/make_golden_p2p_loss_types.py asserts bit-equal to the reference's: the
    same logits give the same g, so the bin counts and acc_sum must be exact."""
    gold = np.load(os.path.join(GOLD, f'p2p_loss_types_{name}.npz'))
    inp, cfg = olt.case_inputs(name)
    head = build(cfg, inp['weights'])
    for step in range(olt.CASES[name].get('steps', 1)):
        inp, _ = olt.case_inputs(name, step)
        with torch.no_grad():
            oc, opo = oml.head_forward(inp['xs'], inp['weights'], cfg)
        cm = [c.cuda().requires_grad_(True) for c in oc]
        pm = [p.cuda().requires_grad_(True) for p in opo]
        losses = head.loss(cm, pm, *_loss_args(inp))
        (sum(losses['loss_cls']) + sum(losses['loss_pts'])).backward()
        for k in ('loss_cls', 'loss_pts'):
            _close(_stack(losses[k]), gold[f'{k}/{step}'], 1e-4, f'{name} step {step} {k}')
        for kind in ('cls', 'reg'):
            if f'{kind}_counts/{step}' in gold.files:
                assert np.array_equal(head._last_ghm[f'{kind}_counts'].cpu().numpy(), gold[f'{kind}_counts/{step}']), (name, step, kind)
        for k in ('loss_cls.acc_sum', 'loss_reg.acc_sum'):
            if f'{k}/{step}' in gold.files:
                assert np.array_equal(head.state_dict()[k].cpu().numpy(), gold[f'{k}/{step}']), (name, step, k)
    for l in range(len(cm)):
        _close(cm[l].grad.cpu().numpy(), gold[f'dmap_cls/{l}'], 1e-4, f'{name} d/dcls_out[{l}]')
        _close(pm[l].grad.cpu().numpy(), gold[f'dmap_pts/{l}'], 1e-4, f'{name} d/dpts_out[{l}]')


def _safe(name):
    """no GHMC g of the case within SAFE_MARGIN of a bin edge: the device's own logits (within ~1e-6) keep every bin decision."""
    g = np.load(os.path.join(GOLD, f'p2p_loss_types_{name}.npz'))
    return all(float(g[k]) >= olt.SAFE_MARGIN for k in g.files if k.startswith('cls_margin'))


@pytest.mark.parametrize('name', sorted(n for n in olt.CASES if _safe(n)))
def test_training_step_matches_reference(ops, name):
    gold = np.load(os.path.join(GOLD, f'p2p_loss_types_{name}.npz'))
    inp, cfg = olt.case_inputs(name)
    head = build(cfg, inp['weights'])
    for step in range(olt.CASES[name].get('steps', 1)):
        inp, _ = olt.case_inputs(name, step)
        head.zero_grad(set_to_none=True)
        losses = head.forward_train([x.cuda() for x in inp['xs']], inp['img_metas'], *_loss_args(inp)[:2])
        (sum(losses['loss_cls']) + sum(losses['loss_pts'])).backward()
        for k in ('loss_cls', 'loss_pts'):
            _close(_stack(losses[k]), gold[f'{k}/{step}'], 1e-4, f'{name} step {step} {k}')
    assert np.array_equal(head._last_assign['gt_inds'].cpu().numpy().astype(np.int32), gold['gt_inds'])
    for k, p in head.named_parameters():
        step = GRAD_STEP if p.dim() == 4 else 1
        g, ref_ = p.grad.flatten()[::step].double().cpu().numpy(), gold[f'grad/{k}'].astype(np.float64)
        rel = float(np.linalg.norm(g - ref_) / max(np.linalg.norm(ref_), 1e-30))
        print(f'[{name}] d/d{k}: norm-relative error {rel:.2e}')
        if k.startswith(('cls_out', 'reg_out')):
            _close(g, ref_, 1e-4, f'{name} d/d{k}')
        else:
            # tests/test_gpu_p2p_multilevel.py: eight GroupNorm + ReLU layers make the towers' gradients this sensitive to rounding
            assert rel <= (3e-2 if k.startswith('reg_convs') else 5e-3), f'{name} d/d{k}: norm-relative error {rel:.3e}'


def _step(head, xs, inp):
    head.zero_grad(set_to_none=True)
    outs = head(xs)
    losses = head.loss(*outs, *_loss_args(inp))
    (sum(losses['loss_cls']) + sum(losses['loss_pts'])).backward()
    return outs, losses


def test_deterministic_repeat(ops):
    """two fresh heads, the same inputs, GHMC with momentum + GHMR over two levels: losses, gradients and acc_sum bit for bit."""
    name = 'two_level_ghm'
    inp, cfg = olt.case_inputs(name)
    cfg['loss_cls_cfg'] = dict(cfg['loss_cls_cfg'], momentum=0.75)
    cfg['loss_reg_cfg'] = dict(cfg['loss_reg_cfg'], momentum=0.75)
    xs = [x.cuda() for x in inp['xs']]
    torch.use_deterministic_algorithms(True)
    try:
        runs = []
        for _ in range(2):
            head = build(cfg, inp['weights'])
            _, losses = _step(head, xs, inp)
            _, losses = _step(head, xs, inp)
            runs.append((losses, {k: p.grad.clone() for k, p in head.named_parameters()},
                         {k: v.clone() for k, v in head.state_dict().items() if 'acc_sum' in k}))
    finally:
        torch.use_deterministic_algorithms(False)
    (l0, g0, a0), (l1, g1, a1) = runs
    for k in ('loss_cls', 'loss_pts'):
        assert np.array_equal(_stack(l0[k]), _stack(l1[k])), k
    assert all(torch.equal(g0[k], g1[k]) for k in g0)
    assert sorted(a0) == ['loss_cls.acc_sum', 'loss_reg.acc_sum'] and all(torch.equal(a0[k], a1[k]) for k in a0)


def _against_oracle_on_own_maps(head, cfg, inp, outs, losses):
    """the oracle on the head's own output maps: the same logits, so the GHMC counts are exact."""
    state = olt.make_state(cfg)
    oc = [c.detach().cpu() for c in outs[0]]
    opo = [p.detach().cpu() for p in outs[1]]
    oloss, aux = olt.p2p_loss(oc, opo, inp['gt_bboxes'], inp['gt_labels'], inp['img_metas'], cfg, state, return_all=True)
    assert np.array_equal(head._last_ghm['cls_counts'].cpu().numpy(), torch.stack(aux['cls_counts']).numpy())
    for k in ('loss_cls', 'loss_pts'):
        _close(_stack(losses[k]), _stack(oloss[k]), 1e-4, k)


def test_ghmc_wide_1203_classes(ops):
    """GHMC(bins=30, momentum=0.75) on a 1203-class single-anchor head: cls_out of 1203 channels runs the column-sliced wide conv."""
    from oracle import p2p_loss_types
    name = 'tinyperson_ghmc'
    inp, cfg = olt.case_inputs(name)
    cfg.update(num_classes=1203, loss_cls_cfg=dict(type='GHMC', bins=30, momentum=0.75, use_sigmoid=True, loss_weight=1.0))
    g = torch.Generator().manual_seed(1203)
    w = oml.weights(g, 1, 1203, False)
    inp['gt_labels'] = [torch.randint(0, 1203, (len(l),), generator=g) for l in inp['gt_labels']]
    inp['xs'] = [x[..., :8, :8].contiguous() for x in inp['xs']]
    head = build(cfg, w)
    assert head.cls_out.out_channels == 1203
    outs, losses = _step(head, [x.cuda() for x in inp['xs']], inp)
    assert p2p_loss_types.CASES[name]['num_classes'] == 1          # the case itself is unchanged
    _against_oracle_on_own_maps(head, cfg, inp, outs, losses)
    assert bool(torch.isfinite(head.cls_out.weight.grad).all()) and float(head.cls_out.weight.grad.abs().max()) > 0


def test_fp16_feature_map(ops):
    """an fp16 FPN map (an autocast backbone's output) into the GHMC + GHMR head: the towers take it as it is."""
    name = 'two_level_ghm'
    inp, cfg = olt.case_inputs(name)
    head = build(cfg, inp['weights'])
    outs, losses = _step(head, [x.cuda().half() for x in inp['xs']], inp)
    assert head.last_input_path == 'fp16-direct', head.last_input_path
    _against_oracle_on_own_maps(head, cfg, inp, outs, losses)
    assert all(bool(torch.isfinite(p.grad).all()) for p in head.parameters())
