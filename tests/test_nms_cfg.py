"""CPU: the one reading of an mmcv nms config (post_processing.parse_nms_cfg) and the one NMS dispatch (run_multiclass_nms) the heads
share.  The NMS ops are replaced by recorders, so each head's kernel choice and arguments are checked without a GPU; the kernels
themselves are tested in tests/test_gpu_nms.py and tests/test_gpu_multiclass_nms_roi.py."""
import inspect

import numpy as np
import pytest
import torch

from oracle import roi_head as orh
from oracle import rpn_loss as orl
from pointtinybenchmark_b200 import ops, post_processing, tile_test
from pointtinybenchmark_b200.p2p_head import P2PHead
from pointtinybenchmark_b200.roi_head import StandardRoIHead
from pointtinybenchmark_b200.registry import CfgNode
from pointtinybenchmark_b200.rpn import RPNProposals


class FakeCuda(torch.Tensor):
    """a CPU tensor that reports is_cuda: lets the CUDA-only guards pass in this dry run"""
    is_cuda = property(lambda s: True)


def fc(t):
    return t.as_subclass(FakeCuda)


def rec(kind, iou, split_thr=10000, agnostic=False, sigma=0.5, min_score=1e-3, method='linear'):
    return post_processing.NmsCfg(kind, iou, sigma, min_score, method, agnostic, split_thr)


PARSE_CASES = [      # (nms cfg, default_iou, the record or the exception)
    (dict(type='nms', iou_threshold=0.6), None, rec('nms', 0.6)),
    (dict(type='nms', iou_thr=0.4), None, rec('nms', 0.4)),
    (dict(type='nms', iou_threshold=0.6, iou_thr=0.4), None, rec('nms', 0.6)),
    (dict(iou_threshold=0.6), None, rec('nms', 0.6)),
    (dict(type='nms'), None, KeyError),
    (dict(type='nms'), 0.5, rec('nms', 0.5)),
    (dict(), 0.7, rec('nms', 0.7)),
    (dict(type='nms', iou_thr=0.4), 0.5, rec('nms', 0.4)),
    (dict(type='soft_nms'), None, rec('soft_nms', 0.3)),
    (dict(type='soft_nms'), 0.5, rec('soft_nms', 0.5)),
    (dict(type='soft_nms', iou_thr=0.45), None, rec('soft_nms', 0.45)),
    (dict(type='soft_nms', iou_threshold=0.4, sigma=0.7, min_score=0.01, method='gaussian'), None,
     rec('soft_nms', 0.4, sigma=0.7, min_score=0.01, method='gaussian')),
    (dict(type='soft_nms', iou_threshold=0.4, method='naive'), None, rec('soft_nms', 0.4, method='naive')),
    (dict(type='soft_nms', iou_threshold=0.4, method='linear'), None, rec('soft_nms', 0.4)),
    (dict(type='nms', iou_threshold=0.5, split_thr=10000), None, rec('nms', 0.5)),
    (dict(type='nms', iou_threshold=0.5, split_thr=5000), None, rec('nms', 0.5, split_thr=5000)),
    (dict(type='nms', iou_threshold=0.5, class_agnostic=True), None, rec('nms', 0.5, agnostic=True)),
    (dict(type='nms', iou_threshold=0.5, unknown=1), None, rec('nms', 0.5)),
    (dict(type='batched_nms', iou_threshold=0.5), None, NotImplementedError),
    (dict(type='soft_nms', iou_threshold=0.5, foo=3), 0.5, rec('soft_nms', 0.5)),
]


@pytest.mark.parametrize('cfg,default_iou,want', PARSE_CASES)
def test_parse_nms_cfg(cfg, default_iou, want):
    if isinstance(want, type):
        with pytest.raises(want):
            post_processing.parse_nms_cfg(cfg, default_iou)
    else:
        assert post_processing.parse_nms_cfg(cfg, default_iou) == want


def test_keep_limit_and_check_kept():
    assert post_processing.keep_limit(-1) == (1024, True) and post_processing.keep_limit(0) == (1024, True)
    assert post_processing.keep_limit(100) == (100, False) and post_processing.keep_limit(1024) == (1024, False)
    with pytest.raises(NotImplementedError):
        post_processing.keep_limit(1025)
    post_processing.check_kept(1023, 1024, True)
    post_processing.check_kept(100, 100, False)
    with pytest.raises(NotImplementedError, match='1023'):
        post_processing.check_kept(1024, 1024, True)


NMS_OPS = ('multiclass_nms', 'multiclass_nms_boxes', 'multiclass_soft_nms')


@pytest.fixture()
def calls(monkeypatch):
    """the NMS ops record (op name, every argument bound to its parameter name, defaults included) and return no detection"""
    log = []

    def recorder(name):
        sig = inspect.signature(getattr(ops, name))

        def op(*args, **kwargs):
            bound = sig.bind(*args, **kwargs)
            bound.apply_defaults()
            log.append((name, dict(bound.arguments)))
            B, k = bound.arguments['scores'].shape[0], bound.arguments['max_per_img']
            return (torch.zeros(B, dtype=torch.int32), torch.zeros(B, k, 5), torch.zeros(B, k, dtype=torch.int32),
                    torch.zeros(B, k, dtype=torch.int32), torch.zeros(B, dtype=torch.int32))
        return op

    for name in NMS_OPS:
        monkeypatch.setattr(ops, name, recorder(name))
    return log


def scalars(args):
    return {k: v for k, v in args.items() if not isinstance(v, torch.Tensor)}


def hard(iou, kmax):
    return 'multiclass_nms_boxes', dict(score_thr=0.05, iou_thr=iou, max_per_img=kmax)


def soft(iou, kmax, sigma=0.5, min_score=1e-3, method='linear'):
    return 'multiclass_soft_nms', dict(pseudo_wh=None, score_thr=0.05, iou_thr=iou, max_per_img=kmax, sigma=sigma, min_score=min_score,
                                       method=method, wide=False)


# (nms cfg, max_per_img, the op and its scalar arguments: those of the code before parse_nms_cfg, with the boxes' default IoU 0.5)
DISPATCH_CASES = [
    (dict(type='nms', iou_threshold=0.6), 100, hard(0.6, 100)),
    (dict(type='nms', iou_thr=0.4), 100, hard(0.4, 100)),
    (dict(type='nms'), 100, hard(0.5, 100)),
    (dict(), -1, hard(0.5, 1024)),
    (dict(type='nms', iou_threshold=0.5, split_thr=10000, unknown=1), 1024, hard(0.5, 1024)),
    (dict(type='soft_nms'), 100, soft(0.5, 100)),
    (dict(type='soft_nms', iou_thr=0.45), 100, soft(0.45, 100)),
    (dict(type='soft_nms', iou_threshold=0.3, sigma=0.7, min_score=0.01, method='gaussian'), 50, soft(0.3, 50, 0.7, 0.01, 'gaussian')),
    (dict(type='soft_nms', iou_threshold=0.3, method='naive'), -1, soft(0.3, 1024, method='naive')),
    (dict(type='nms', iou_threshold=0.5, split_thr=5000), 100, NotImplementedError),
    (dict(type='batched_nms', iou_threshold=0.5), 100, NotImplementedError),
    (dict(type='nms', iou_threshold=0.5), 2000, NotImplementedError),
]


def _boxes(n, C, class_specific):
    g = torch.Generator().manual_seed(n + C)
    c = torch.rand(n, C if class_specific else 1, 2, generator=g) * 200
    return torch.cat([c - 8, c + 8], -1).reshape(n, -1)


@pytest.mark.parametrize('class_specific', [False, True])
@pytest.mark.parametrize('cfg,max_num,want', DISPATCH_CASES)
def test_multiclass_nms_records(calls, cfg, max_num, want, class_specific):
    n, C = 30, 3
    boxes, scores = _boxes(n, C, class_specific), torch.rand(n, C + 1, generator=torch.Generator().manual_seed(1))
    run = lambda: post_processing.multiclass_nms(fc(boxes), fc(scores), 0.05, cfg, max_num)
    if isinstance(want, type):
        with pytest.raises(want):
            run()
        assert calls == []
        return
    run()
    (name, args), = calls
    assert (name, scalars(args)) == want
    geom = args['pts_or_boxes' if name == 'multiclass_soft_nms' else 'boxes']
    assert tuple(geom.shape) == ((1, n, C, 4) if class_specific else (1, n, 4)) and tuple(args['scores'].shape) == (1, n, C)
    assert torch.equal(args['scores'][0].as_subclass(torch.Tensor), scores[:, :C])


@pytest.mark.parametrize('kind', ['nms', 'soft_nms'])
def test_multiclass_nms_class_agnostic_records(calls, kind):
    """class_agnostic: one kernel class over every (box, class) candidate"""
    n, C = 30, 3
    boxes, scores = _boxes(n, C, False), torch.rand(n, C + 1, generator=torch.Generator().manual_seed(1))
    post_processing.multiclass_nms(fc(boxes), fc(scores), 0.05, dict(type=kind, iou_threshold=0.6, class_agnostic=True), 100)
    (name, args), = calls
    assert (name, scalars(args)) == (hard(0.6, 100) if kind == 'nms' else soft(0.6, 100))
    geom = args['pts_or_boxes' if kind == 'soft_nms' else 'boxes']
    assert tuple(geom.shape) == (1, n * C, 4) and tuple(args['scores'].shape) == (1, n * C, 1)


@pytest.mark.parametrize('cfg,max_per_img,want', DISPATCH_CASES + [(None, -1, hard(0.5, 1024)),
                                                                   (dict(type='nms', iou_threshold=0.5, class_agnostic=True), 100,
                                                                    NotImplementedError)])
def test_roi_head_multiclass_nms_records(calls, cfg, max_per_img, want):
    head = StandardRoIHead(**orh.head_kwargs('tinyperson'))
    boxes, scores = fc(torch.rand(2, 30, 3, 4)), fc(torch.rand(2, 30, 3))
    run = lambda: head._multiclass_nms(boxes, scores, CfgNode(score_thr=0.05, nms=cfg, max_per_img=max_per_img))
    if isinstance(want, type):
        with pytest.raises(want):
            run()
        assert calls == []
        return
    out = run()
    (name, args), = calls
    assert (name, scalars(args)) == want
    assert args['pts_or_boxes' if name == 'multiclass_soft_nms' else 'boxes'] is boxes and args['scores'] is scores
    assert out[3:] == (want[1]['max_per_img'], max_per_img <= 0)


# ---- the two behaviour changes: `iou_thr` reaches P2P soft-NMS and the RPN; P2P refuses class_agnostic instead of ignoring it
def _p2p(monkeypatch, nms):
    head = P2PHead(2, 256, point_anchor=[(0., 0.)], strides=[8], test_cfg=dict(nms_pre=-1, score_thr=0.05, nms=nms, max_per_img=100))
    P = 40

    def decode(cmap, rmap, C, *args):
        g = torch.Generator().manual_seed(0)
        return torch.arange(P, dtype=torch.int32)[None], torch.rand(1, P, 2, generator=g) * 64, torch.rand(1, P, C, generator=g)
    monkeypatch.setattr(ops, 'p2p_decode_topk', decode)
    return head


def _p2p_get_bboxes(head):
    return head.get_bboxes([fc(torch.zeros(1, 2, 8, 8))], [fc(torch.zeros(1, 2, 8, 8))], [dict(img_shape=(64, 64, 3))])


def _p2p_aug_test(head):
    head.forward = lambda x: (x, x)
    head.get_bboxes = lambda *a, **kw: [(torch.tensor([[1., 2., 17., 18., 0.9], [30., 30., 46., 46., 0.8]]), torch.tensor([0, 1]))]
    meta = dict(img_shape=(64, 64, 3), scale_factor=np.ones(4, np.float32), flip=False)
    return head.aug_test_bboxes([None], [[meta]])


@pytest.mark.parametrize('site', [_p2p_get_bboxes, _p2p_aug_test])
def test_p2p_soft_nms_honours_iou_thr(calls, monkeypatch, site):
    site(_p2p(monkeypatch, dict(type='soft_nms', iou_thr=0.45, sigma=0.6, method='gaussian')))
    (name, args), = calls
    assert name == 'multiclass_soft_nms' and args['iou_thr'] == 0.45 and (args['sigma'], args['method']) == (0.6, 'gaussian')
    calls.clear()
    site(_p2p(monkeypatch, dict(type='soft_nms')))                   # soft_nms' own default
    assert calls[0][1]['iou_thr'] == 0.3


@pytest.mark.parametrize('site', [_p2p_get_bboxes, _p2p_aug_test])
def test_p2p_hard_nms_records(calls, monkeypatch, site):
    site(_p2p(monkeypatch, dict(type='nms', iou_thr=0.4)))
    (name, args), = calls
    if site is _p2p_get_bboxes:
        assert name == 'multiclass_nms' and args['pseudo_wh'] == (16, 16) and args['wide'] is False
    else:
        assert name == 'multiclass_nms_boxes'
    assert (args['iou_thr'], args['max_per_img']) == (0.4, 100)
    with pytest.raises(KeyError):
        site(_p2p(monkeypatch, dict(type='nms')))


@pytest.mark.parametrize('site', [_p2p_get_bboxes, _p2p_aug_test])
@pytest.mark.parametrize('kind', ['nms', 'soft_nms'])
def test_p2p_refuses_class_agnostic(calls, monkeypatch, site, kind):
    with pytest.raises(NotImplementedError, match='class_agnostic'):
        site(_p2p(monkeypatch, dict(type=kind, iou_threshold=0.5, class_agnostic=True)))
    assert calls == []


@pytest.mark.parametrize('nms,iou,merge_iou', [(dict(type='nms', iou_thr=0.6), 0.6, 0.6), (dict(type='nms', iou_threshold=0.65), 0.65, 0.65),
                                               (dict(type='nms'), 0.7, KeyError), (None, 0.55, 0.55)])
def test_rpn_honours_iou_thr(monkeypatch, nms, iou, merge_iou):
    """the RPN's proposals (default IoU 0.7) and its tile merge (no default); the older `nms_thr` stands for the nms config only
    where that is absent"""
    seen = []
    sig = inspect.signature(ops.rpn_proposals)
    monkeypatch.setattr(ops, 'rpn_proposals', lambda *a: seen.append(sig.bind(*a).arguments['iou_thr']))
    cfg = dict(nms_pre=100, max_per_img=50, min_bbox_size=0, nms_thr=0.55)
    if nms is not None:
        cfg['nms'] = nms
    prop = RPNProposals(orl.TINYPERSON['anchor_generator'], orl.TINYPERSON['bbox_coder'], cfg)
    L = len(orl.STRIDES)
    prop.get_bboxes_padded([fc(torch.zeros(1, 3, 4, 4))] * L, [fc(torch.zeros(1, 12, 4, 4))] * L, [dict(img_shape=(16, 16, 3))])
    assert seen == [iou]
    if merge_iou is KeyError:
        with pytest.raises(KeyError):
            tile_test._rpn_merge_cfg(cfg)
    else:
        assert tile_test._rpn_merge_cfg(cfg) == (merge_iou, 50)
    with pytest.raises(NotImplementedError):
        tile_test._rpn_merge_cfg(dict(nms=dict(type='soft_nms', iou_threshold=0.7), max_per_img=50))


def test_tile_merge_cfg():
    assert tile_test._merge_nms_cfg(dict()) == (0.5, 10000)
    assert tile_test._merge_nms_cfg(dict(nms=dict(type='nms', iou_thr=0.4, split_thr=5000))) == (0.4, 5000)
    with pytest.raises(NotImplementedError, match='options'):
        tile_test._merge_nms_cfg(dict(nms=dict(type='nms', iou_threshold=0.5, sigma=0.5)))
