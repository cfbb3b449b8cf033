"""CPU: host-side logic of the plugin layer (registry, ctor/config surface, state_dict keys, CSR builders, Hungarian
driver) and the 'no CPU fallback' rule."""
import os

import numpy as np
import pytest
import torch

from oracle import cpr as ocpr
from pointtinybenchmark_b200 import ops
from pointtinybenchmark_b200.cpr_head import CPRHead, _BatchGT
from pointtinybenchmark_b200.p2p_head import P2PHead
from pointtinybenchmark_b200.registry import HEADS, build_head
from tests.test_gpu_cpr_head import head_cfg as cpr_cfg
from tests.test_gpu_p2p import head_cfg as p2p_cfg

D = dict(num_classes=80, C=256, stride=8, radius=8)


def test_registry_builds_heads_from_reference_style_config_dicts():
    assert HEADS.get('CPRHead') is CPRHead and HEADS.get('P2PHead') is P2PHead
    h = build_head(cpr_cfg(D))
    keys = set(h.state_dict())
    for i in range(4):
        assert {f'cls_convs.{i}.conv.weight', f'cls_convs.{i}.gn.weight', f'cls_convs.{i}.gn.bias'} <= keys
    assert {'cls_out.weight', 'cls_out.bias', 'ins_out.weight', 'ins_out.bias'} <= keys
    assert h.cls_out.weight.shape == (80, 256)
    assert abs(float(h.cls_out.bias[0]) + np.log(99.0)) < 1e-6           # bias_prob=0.01 (cpr_head.py:947)
    p = build_head(p2p_cfg(dict(D, stride=4)))
    pk = set(p.state_dict())
    assert {'cls_out.weight', 'reg_out.weight', 'cls_convs.3.gn.bias', 'reg_convs.0.conv.weight'} <= pk
    assert p.cls_out.weight.shape == (80, 256, 3, 3) and p.reg_out.weight.shape == (2, 256, 3, 3)


def test_unsupported_configurations_fail_loudly():
    bad = cpr_cfg(D); bad['strides'] = [8, 16]
    with pytest.raises(NotImplementedError):
        build_head(bad)
    bad = cpr_cfg(D); bad['ins_share_head_feat'] = False
    with pytest.raises(NotImplementedError):
        build_head(bad)
    bad = cpr_cfg(D); bad['normal_cfg'] = dict(prob_cls_type='sigmoid', out_bg_cls=True)
    with pytest.raises(NotImplementedError):
        build_head(bad)
    var = cpr_cfg(D); var['num_cls_fcs'] = 2; var['fc_out_channels'] = 64; var['loss_mil'] = dict(var['loss_mil'], binary_ins=True)
    hv = build_head(var)          # variants the reference class accepts: built (generic path), with the reference's parameter names / shapes
    assert hv.cls_fcs[1].weight.shape == (64, 64) and hv.cls_out.weight.shape == (80, 64) and hv.ins_out.weight.shape == (160, 64)
    bad = cpr_cfg(D); bad['train_pts_extractor']['pos_generator'] = dict(type='GridEllipsePtFeatGenerator', a_minus_c=2.0)
    with pytest.raises(NotImplementedError):
        build_head(bad)          # (the reference's own implementation of this generator cannot run, DESIGN.md §8)
    ok = cpr_cfg(D); ok['train_pts_extractor']['pos_generator'] = dict(type='GridCirclesPtFeatGenerator', radius=3)
    assert build_head(ok).train_pts_extractor['pos_generator']['type'] == 'GridCirclesPtFeatGenerator'
    with pytest.raises(TypeError):
        build_head(dict(cpr_cfg(D), bogus_kwarg=1))


def test_no_cpu_fallback():
    h = build_head(cpr_cfg(D))
    x = torch.zeros(1, 256, 8, 8)
    gtb, gtl = [torch.tensor([[8., 8., 24., 24.]])], [torch.tensor([3])]
    metas = [dict(pad_shape=(64, 64, 3), img_shape=(64, 64, 3), scale_factor=[1, 1, 1, 1])]
    with pytest.raises(RuntimeError, match='no CPU'):
        h.loss([x], [x], gtb, gtl, metas)
    with pytest.raises(RuntimeError, match='no CPU'):
        h.get_bboxes([x], [x], metas, gt_bboxes=gtb, gt_labels=gtl, gt_anns_id=[torch.tensor([0])])
    with pytest.raises(RuntimeError, match='CUDA'):
        ops.bag_gather(torch.zeros(1, 8, 8, 4), torch.zeros(1, 2), torch.zeros(1, dtype=torch.int32), torch.zeros(1, 2), 8,
                       torch.zeros(1, 2, dtype=torch.int32))


def test_offset_table_is_bit_identical_to_the_reference_formula():
    for r, s in [(5, 8), (8, 8), (8, 4), (3, 16)]:
        off = ops.circle_offsets(r, s)
        ref = torch.cat([ocpr.circle_offsets(r, s), torch.zeros(1, 2)])
        assert torch.equal(off, ref)
        assert off.shape[0] == 8 * r * (r + 1) // 2 + 1


def test_batch_gt_and_label_groups():
    gtb = [torch.tensor([[0., 0., 16., 16.], [10., 10., 26., 26.], [4., 4., 20., 20.]]), torch.tensor([[30., 30., 46., 46.]])]
    gtl = [torch.tensor([5, 2, 5]), torch.tensor([5])]
    metas = [dict(pad_shape=(64, 96, 3), img_shape=(60, 90, 3)), dict(pad_shape=(64, 96, 3), img_shape=(61, 91, 3))]
    gt = _BatchGT(gtb, gtl, metas, torch.device('cpu'))
    assert gt.lens == [3, 1] and gt.G == 4
    assert gt.bag_img.tolist() == [0, 0, 0, 1] and gt.img_ptr.tolist() == [0, 3, 4]
    assert gt.pad_hw.tolist() == [[64, 96], [64, 96]] and gt.img_hw.tolist() == [[60, 90], [61, 91]]
    assert torch.equal(gt.centers, torch.tensor([[8., 8.], [18., 18.], [12., 12.], [38., 38.]]))
    grp_of, grp_ptr, grp_idx = ops.label_groups(gt.bag_img, gt.labels, 80)
    groups = {}
    for g in range(4):
        a, b = int(grp_ptr[grp_of[g]]), int(grp_ptr[grp_of[g] + 1])
        groups[g] = grp_idx[a:b].tolist()
    assert groups == {0: [0, 2], 2: [0, 2], 1: [1], 3: [3]}       # same (image,label), ascending GT order
    with pytest.raises(NotImplementedError):
        _BatchGT([torch.zeros(4, 4)], [torch.tensor([1, 2])], metas[:1], torch.device('cpu'))   # num_refine = 2


def test_every_shipped_cpr_p2p_config_builds(golden_dir):
    """"drops into the existing configs unchanged": the bbox_head dicts of every CPR / P2P config under the reference's
    configs2/ (extracted by oracle/make_cfg_fixture.py) build this package's heads; the two entries the reference itself
    cannot run (CascadeCPRHead is not in its tree; a config whose _base_ file is missing) are the only exceptions."""
    import json
    import os
    cfgs = json.load(open(os.path.join(golden_dir, 'reference_head_cfgs.json')))
    built = 0
    for name, c in cfgs.items():
        if 'error' in c:
            assert 'FileNotFoundError' in c['error']          # broken in the reference too
            continue
        head_cfg = dict(c['bbox_head'])
        if head_cfg['type'] == 'CascadeCPRHead':              # unreleased (SURVEY.md §0)
            with pytest.raises(KeyError):
                build_head(head_cfg)
            continue
        head = build_head(head_cfg, default_args=dict(train_cfg=c.get('train_cfg'), test_cfg=c.get('test_cfg')))
        assert type(head).__name__ == head_cfg['type']
        assert head.strides == list(head_cfg['strides']) and head.num_classes == head_cfg['num_classes']
        built += 1
    assert built >= 13


def test_api_signatures_match_reference(golden_dir):
    """every parameter of the reference's plugin classes / functions on the path (recorded from the real reference by
    oracle/make_golden.py::golden_api_signatures) is accepted by the mirror, in the same relative order."""
    import inspect
    import json
    from pointtinybenchmark_b200 import assigners, dist, post_processing, rpn
    from pointtinybenchmark_b200.cpr_head import CPRHead
    ref = json.load(open(os.path.join(golden_dir, 'api_signatures.json')))
    ours = {'CPRHead': CPRHead, 'P2PHead': P2PHead, 'MaxIoUAssigner': assigners.MaxIoUAssigner, 'PointAssigner': assigners.PointAssigner,
            'HungarianAssignerV2': assigners.HungarianAssignerV2, 'PseudoSampler': assigners.PseudoSampler, 'AnchorGenerator': rpn.AnchorGenerator}
    funcs = {'multiclass_nms': post_processing.multiclass_nms, 'RPNHead.get_bboxes': rpn.RPNProposals.get_bboxes,
             'BaseDetector._parse_losses': dist.parse_losses}
    checked = 0
    for key, want in ref.items():
        if key in funcs:
            f = funcs[key]
        else:
            cls, m = key.split('.')
            f = getattr(ours[cls], m)
        have = [p.name for p in inspect.signature(f).parameters.values() if p.name != 'self' and p.kind not in (p.VAR_KEYWORD, p.VAR_POSITIONAL)]
        assert [n for n in want if n not in have] == [], (key, want, have)
        assert [n for n in have if n in want] == want, (key, 'order')
        checked += 1
    assert checked == len(ref) >= 25


def test_state_dict_matches_reference_for_every_shipped_config(golden_dir):
    """checkpoint compatibility (`load_state_dict(strict=True)` of cpr_epoch_12.pth / p2p checkpoints): the mirror built from each shipped
    CPR / P2P config exposes EXACTLY the parameter / buffer names and shapes of the real reference head (recorded by
    oracle/make_golden.py::golden_state_dict_keys)."""
    import json
    cfgs = json.load(open(os.path.join(golden_dir, 'reference_head_cfgs.json')))
    ref = json.load(open(os.path.join(golden_dir, 'state_dict_shapes.json')))
    assert len(ref) >= 13
    for name, want in ref.items():
        c = cfgs[name]
        head = build_head(dict(c['bbox_head']), default_args=dict(train_cfg=c.get('train_cfg'), test_cfg=c.get('test_cfg')))
        have = {k: list(v.shape) for k, v in head.state_dict().items()}
        assert have == want, (name, sorted(set(have) ^ set(want))[:6])


def test_packed_weight_caches_are_invalidated_by_train_eval_and_load_state_dict():
    """ADVICE r1: the tensor-core packings are keyed on Tensor._version, which `.data` writes (EMA swaps, weight surgery) do not bump.
    The heads drop the caches on train() / eval(), after load_state_dict (also when loaded as a SUBMODULE of a detector) and on demand."""
    from pointtinybenchmark_b200.fcos_head import FCOSHead
    from pointtinybenchmark_b200.layers import _PACK_ATTRS
    fcos = FCOSHead(num_classes=80, in_channels=256)
    for h, mods in ((build_head(cpr_cfg(D)), 'cls_convs.0 cls_convs.3 cls_out'),
                    (build_head(p2p_cfg(dict(D, stride=4))), 'cls_convs.0 cls_convs.3 cls_out'),
                    (fcos, 'cls_convs.0 reg_convs.3 conv_cls conv_reg conv_centerness')):
        mods = [h.get_submodule(n) for n in mods.split()]

        def plant():
            for m in mods:
                for a in _PACK_ATTRS:
                    setattr(m, a, ('stale-key', 'stale-pack'))

        def clean():
            return not any(hasattr(m, a) for m in h.modules() for a in _PACK_ATTRS)
        plant(); h.eval(); assert clean(), 'eval()'
        plant(); h.train(); assert clean(), 'train()'
        plant(); h.load_state_dict(h.state_dict()); assert clean(), 'load_state_dict on the head'
        det = torch.nn.Module()
        det.bbox_head = h
        plant(); det.load_state_dict(det.state_dict()); assert clean(), 'load_state_dict on an enclosing detector'
        plant(); h.invalidate_packed(); assert clean(), 'explicit invalidate_packed()'


def test_batch_gt_index_arrays_are_cached_per_shape():
    from pointtinybenchmark_b200 import cpr_head as ch
    ch._GT_INDEX_CACHE.clear()
    metas = [dict(pad_shape=(64, 96, 3), img_shape=(60, 90, 3))] * 2
    mk = lambda n: (torch.rand(n, 4), torch.zeros(n, dtype=torch.long))
    (b0, l0), (b1, l1) = mk(3), mk(5)
    g1 = _BatchGT([b0, b1], [l0, l1], metas, torch.device('cpu'))
    g2 = _BatchGT([b0 + 1, b1 + 1], [l0, l1], metas, torch.device('cpu'))
    assert len(ch._GT_INDEX_CACHE) == 1 and g1.bag_img.data_ptr() == g2.bag_img.data_ptr(), 'same lens / metas: no new upload'
    assert g1.bag_img.tolist() == [0, 0, 0, 1, 1, 1, 1, 1] and g1.img_ptr.tolist() == [0, 3, 8]
    assert g1.pad_hw.tolist() == [[64, 96]] * 2 and g1.img_hw.tolist() == [[60, 90]] * 2
    _BatchGT([b1, b0], [l1, l0], metas, torch.device('cpu'))
    assert len(ch._GT_INDEX_CACHE) == 2
