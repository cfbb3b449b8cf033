"""CPU: the tile-testing restatement (oracle/tile_test.py) — ATen's CPU summation order of merge_aug_bboxes' stack-mean, the box
mappings, the tile grouping and the refusals of StandardRoIHead.aug_test / tile_aug_test."""
import numpy as np
import pytest
import torch

from oracle import roi_head as orh
from oracle import tile_test as ott


@pytest.mark.parametrize('A', list(range(1, 18)) + [31, 33, 63])
@pytest.mark.parametrize('M', [8, 12, 31, 32, 33, 100, 1028, 4000, 4004])
def test_aten_mean_order(A, M):
    """torch.stack(...).mean(0) on the CPU equals the restated order bit for bit (the order ptb_aug_merge uses) for stacks of at least
    8 columns; narrower stacks (a tile of one proposal) reduce in an order that is not restated"""
    g = np.random.default_rng(A * 1000 + M)
    x = (g.standard_normal((A, M)) * g.random((A, M)) * 1000).astype(np.float32)
    assert np.array_equal(torch.from_numpy(x).mean(0).numpy(), ott.aten_mean0(x))


@pytest.mark.parametrize('direction', ['horizontal', 'vertical', 'diagonal'])
def test_mapping_round_trip(direction):
    g = torch.Generator().manual_seed(3)
    b = torch.rand(50, 4, generator=g) * 200
    b[:, 2:] += b[:, :2]
    m = dict(img_shape=(600, 800, 3), scale_factor=np.array([1.5, 1.5, 1.5, 1.5], np.float32), flip=True, flip_direction=direction)
    assert torch.allclose(ott.bbox_mapping_back(ott.bbox_mapping(b, m), m), b, atol=1e-4)


def test_tile_mapping_drops_and_clamps():
    b = torch.tensor([[10., 10., 50., 50.], [100., 100., 101., 140.], [-30., 5., 20., 30.]])
    m = dict(img_shape=(64, 64, 3), scale_factor=np.ones(4, np.float32), flip=False, tile_offset=(5, 0))
    out = ott.bbox_mapping(b, m)
    assert out.tolist() == [[5., 10., 45., 50.], [0., 5., 15., 30.]]


def test_group_tiles_pops_offsets_in_first_appearance_order():
    from pointtinybenchmark_b200.tile_test import group_tiles
    metas = [[dict(tile_offset=o, k=i)] for i, o in enumerate([(0, 0), (100, 0), (0, 0), (100, 0), (0, 50)])]
    assert group_tiles(metas) == [((0, 0), [0, 2]), ((100, 0), [1, 3]), ((0, 50), [4])]
    assert all('tile_offset' not in m[0] for m in metas)


def test_refusals():
    from pointtinybenchmark_b200.roi_head import StandardRoIHead
    from pointtinybenchmark_b200 import tile_test
    h = StandardRoIHead(**orh.head_kwargs('tinyperson'), test_cfg=dict(orh.TEST, do_tile_as_aug=True))
    with pytest.raises(NotImplementedError, match='do_tile_as_aug'):
        h.aug_test(None, None, None)
    with pytest.raises(NotImplementedError, match='soft-NMS'):
        tile_test._merge_nms_cfg(dict(nms=dict(type='soft_nms', iou_threshold=0.5)))
    with pytest.raises(NotImplementedError, match='class_agnostic'):
        tile_test._merge_nms_cfg(dict(nms=dict(type='nms', iou_threshold=0.5, class_agnostic=True)))
    assert tile_test._rpn_merge_cfg(dict(nms=dict(type='nms', iou_threshold=0.7), max_num=300)) == (0.7, 300)
