"""CPU: CPRHead above 256 classes — the oracle against the golden vectors recorded from the REAL reference at 365 and 1203 classes
(oracle/make_golden_cpr_many_classes.py), and the host restatement of the chunked MIL forward (tests/mil_chunk_ref.py) against float64."""
import os

import numpy as np
import pytest
import torch

from oracle import cpr as ocpr
from oracle.make_golden_cpr_many_classes import CLASS_COUNTS, many_class_inputs, oracle_cfg
from tests.mil_chunk_ref import mil_fwd_chunked, mil_lanes, mil_ref64

EPS = 1e-6


@pytest.mark.parametrize('N', CLASS_COUNTS)
def test_oracle_matches_reference_golden(golden_dir, N):
    gold = np.load(os.path.join(golden_dir, f'cpr_many_classes_{N}.npz'))
    inp = many_class_inputs(N, int(gold['seed']))
    cfg = oracle_cfg(inp['cfgd'])
    w = inp['weights']
    f = inp['cls_feat'].clone().requires_grad_(True)
    wo = {k: v.clone().requires_grad_(True) for k, v in w.items()}
    ol, oall = ocpr.cpr_loss(f, wo, inp['gt_bboxes'], inp['gt_labels'], inp['img_metas'], cfg, return_all=True)
    sum(v for k, v in ol.items() if 'loss' in k).backward()
    for k in ('gt_loss', 'pos_loss', 'neg_loss', 'bag_acc'):
        np.testing.assert_allclose(ol[k].detach().reshape(-1).numpy(), gold['loss_' + k], rtol=1e-6, atol=1e-7, err_msg=k)
    sub = f.grad.flatten()[::211].numpy()
    assert np.abs(sub - gold['grad_feat_sub']).max() <= 1e-6 * max(1.0, np.abs(gold['grad_feat_sub']).max())
    for name, key in (('cls_out.weight', 'grad_cls_w'), ('cls_out.bias', 'grad_cls_b'), ('ins_out.weight', 'grad_ins_w'),
                      ('ins_out.bias', 'grad_ins_b')):
        np.testing.assert_allclose(wo[name].grad.numpy(), gold[key], rtol=0, atol=1e-6 * max(1.0, np.abs(gold[key]).max()), err_msg=name)
    np.testing.assert_allclose(oall['bag_prob'].detach().numpy(), gold['mil_bag_prob'], rtol=0, atol=1e-7)
    valid = gold['pos_valid'].reshape(len(gold['pos_valid']), -1)
    assert valid[-1].any() and not valid[-1].all(), 'the edge GT has a bag partly outside pad_shape'
    with torch.no_grad():
        res, rall = ocpr.cpr_get_bboxes(inp['cls_feat'], w, inp['gt_bboxes'], inp['gt_labels'], inp['gt_anns_id'], inp['img_metas'], cfg,
                                        return_all=True)
    np.testing.assert_array_equal(torch.cat([r[0] for r in res]).numpy(), gold['det'])
    np.testing.assert_array_equal(torch.cat([r['chosen'] for r in rall['refine']]).numpy(), gold['chosen'])
    np.testing.assert_array_equal(torch.cat([r['not_refine'] for r in rall['refine']]).numpy(), gold['not_refine'])


def _bags(N, K, seed, G=5):
    """bag logits (G,K,LD) with LD = 2 ceil8(N), pad columns 50; bag 0 has no valid sample, the others about 70 %."""
    g = torch.Generator().manual_seed(seed)
    NP = (N + 7) // 8 * 8
    bl = torch.full((G, K, 2 * NP), 50.0)
    bl[..., :N] = torch.randn(G, K, N, generator=g) * 2.0 - 1.0
    bl[..., NP:NP + N] = torch.randn(G, K, N, generator=g) * 2.0
    weight = (torch.rand(G, K, generator=g) < 0.7).float()
    weight[0] = 0.0
    weight[1:, -1] = 1.0
    labels = torch.randint(0, N, (G,), generator=g)
    return bl, NP, weight, labels


@pytest.mark.parametrize('kind', [0, 1])
@pytest.mark.parametrize('N,K', [(257, 33), (365, 9), (513, 1)])
def test_chunked_restatement_matches_float64(N, K, kind):
    bl, NP, weight, labels = _bags(N, K, 100 * N + K + kind)
    prob, loss, lw, top = mil_fwd_chunked(bl.numpy(), N, NP, weight.numpy(), labels.numpy(), EPS, kind)
    ref = mil_ref64(bl, N, NP, weight, labels, EPS, kind)
    assert np.abs(prob - ref['prob'].numpy()).max() <= 1e-5 * max(1.0, float(ref['prob'].abs().max()))
    assert abs(float(loss.astype(np.float64).sum()) - ref['sum']) <= 2e-5 * max(1.0, abs(ref['sum']))
    assert float(lw.sum()) == ref['count']
    close = ref['margin'].numpy() <= 1e-5
    hits = top == labels.numpy()
    ref_hits = (ref['prob'].argmax(dim=1) == labels).numpy()
    assert np.array_equal(hits[~close], ref_hits[~close])


@pytest.mark.parametrize('N', [257, 600])
def test_chunk_width_does_not_change_class_values(N):
    """every per-(bag, class) value is formed in the same order whatever the chunk width: probabilities are bit-identical."""
    bl, NP, weight, labels = _bags(N, 33, N)
    base = mil_fwd_chunked(bl.numpy(), N, NP, weight.numpy(), labels.numpy(), EPS, 0)
    for cp in (32, 96, 128):
        other = mil_fwd_chunked(bl.numpy(), N, NP, weight.numpy(), labels.numpy(), EPS, 0, cp=cp)
        assert np.array_equal(base[0], other[0]) and np.array_equal(base[3], other[3])
    assert mil_lanes(N) == 256 and mil_lanes(200) == 224 and mil_lanes(9) == 32


def test_top1_tie_across_a_chunk_boundary_takes_the_first_class():
    """classes 255 and 256 (chunks 0 and 1) hold identical logits and the largest bag probability: the first maximum, 255, is the top-1."""
    N = 300
    bl, NP, weight, labels = _bags(N, 9, 7, G=2)
    for c in (255, 256):
        bl[..., c] = 6.0
        bl[..., NP + c] = 0.5
    for lab, hit in ((255, True), (256, False)):
        labels[:] = lab
        _, _, _, top = mil_fwd_chunked(bl.numpy(), N, NP, weight.numpy(), labels.numpy(), EPS, 0)
        assert top[1] == 255 and (top[1] == lab) == hit
