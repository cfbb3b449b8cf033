"""CPU: oracle/fcos.py against the reference's FCOS fixtures (tests/golden/fcos_*.npz, written by oracle/make_golden_fcos.py), the
reference's constructor keywords and state_dict names / shapes against FCOSHead's, and reduce_mean_ over two gloo ranks."""
import inspect
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import fcos as ofc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, 'tests', 'golden')


def gold(name):
    return np.load(os.path.join(GOLD, f'fcos_{name}.npz'))


def maps(name):
    g = gold(name)
    if 'train_cls0' in g:
        return tuple([torch.from_numpy(g[f'{k}_{n}{l}']) for l in range(5)] for n in ('cls', 'reg', 'ctr')
                     for k in ('train',)), tuple([torch.from_numpy(g[f'eval_{n}{l}']) for l in range(5)] for n in ('cls', 'reg', 'ctr'))
    m = ofc.case_inputs(name)['maps']
    return m, m


@pytest.mark.parametrize('name', ['tinyperson', 'coco80', 'options', 'no_pos'])
def test_oracle_targets_and_losses(name):
    g, inp = gold(name), ofc.case_inputs(name)
    cfg = dict(ofc.CASES[name]['head'], stacked_convs=4)
    train, _ = maps(name)
    train = tuple([t.clone().requires_grad_(True) for t in ts] for ts in train)
    losses, tg = ofc.loss(*train, inp['gt_bboxes'], inp['gt_labels'], cfg)
    for l in range(5):
        assert torch.equal(tg['labels'][l], torch.from_numpy(g[f'labels{l}'].astype(np.int64)))
        assert torch.equal(tg['bbox_targets'][l], torch.from_numpy(g[f'bbox_targets{l}']))
    for k, v in losses.items():
        assert abs(float(v) - float(g[k])) <= 1e-6 * max(1.0, abs(float(g[k]))), k
    sum(losses.values()).backward()
    for n, ts in zip(('cls', 'reg', 'ctr'), train):
        for l, t in enumerate(ts):
            if f'grad_{n}{l}' in g:
                assert float((t.grad - torch.from_numpy(g[f'grad_{n}{l}'])).abs().max()) <= 1e-6 * max(1.0, float(np.abs(g[f'grad_{n}{l}']).max()))


@pytest.mark.parametrize('name', ['tinyperson', 'coco80', 'options', 'no_pos'])
def test_oracle_get_bboxes(name):
    g, inp = gold(name), ofc.case_inputs(name)
    c = ofc.CASES[name]
    _, ev = maps(name)
    res, tk = ofc.get_bboxes(*ev, inp['img_metas'], dict(c['head']), c['test'], c.get('rescale', False))
    for b, (d, l) in enumerate(res):
        assert torch.equal(d, torch.from_numpy(g[f'dets{b}']))
        assert torch.equal(l, torch.from_numpy(g[f'det_labels{b}'].astype(np.int64)))
    for l, t in enumerate(tk):
        if t is not None:
            assert torch.equal(t.int(), torch.from_numpy(g[f'topk{l}']))


@pytest.mark.parametrize('name', ['tiles', 'flip_scale'])
def test_oracle_aug_test(name):
    g = gold(name)
    augs = ofc.tile_case(name)
    d, l, rows = ofc.aug_test_bboxes([ofc.aug_maps(a) for a in augs], [[a['meta']] for a in augs], ofc.TINY, ofc.TINY_TEST)
    assert rows == int(g['rows'])
    assert torch.equal(d, torch.from_numpy(g['dets_rescale0']))
    assert torch.equal(l, torch.from_numpy(g['labels_rescale0'].astype(np.int64)))


@pytest.mark.parametrize('name', ['tinyperson', 'coco80'])
def test_state_dict_and_signature_parity(name):
    from pointtinybenchmark_b200.fcos_head import FCOSHead
    g = gold(name)
    head = FCOSHead(**ofc.head_kwargs(name))
    sd = head.state_dict()
    assert sorted(sd) == g['state_keys'].tolist()
    assert [list(sd[k].shape) + [-1] * (4 - sd[k].dim()) for k in sorted(sd)] == g['state_shapes'].tolist()
    head.load_state_dict({k: v for k, v in ofc.case_inputs(name)['weights'].items()}, strict=True)
    params = set(inspect.signature(FCOSHead.__init__).parameters)
    assert set(g['ctor_params'].tolist()) <= params
    assert abs(float(head.conv_cls.bias[0]) - float(-np.log(99.0))) < 1e-6


WORKER = r'''
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1])
from pointtinybenchmark_b200.dist import reduce_mean_
rank = int(os.environ['RANK'])
dist.init_process_group('gloo')
t = torch.tensor([3.0 + rank, 0.5 * (rank + 1)])
reduce_mean_(t)
print(t.tolist())
dist.destroy_process_group()
'''


def test_reduce_mean_two_ranks(tmp_path):
    s = socket.socket(); s.bind(('127.0.0.1', 0)); port = s.getsockname()[1]; s.close()
    w = tmp_path / 'worker.py'
    w.write_text(WORKER)
    procs = [subprocess.Popen([sys.executable, str(w), ROOT], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True,
                              env=dict(os.environ, RANK=str(r), WORLD_SIZE='2', MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port)))
             for r in range(2)]
    outs = [p.communicate(timeout=300) for p in procs]
    assert all(p.returncode == 0 for p in procs), outs
    for o in outs:
        assert eval(o[0].strip().splitlines()[-1]) == [3.5, 0.75]          # (3 + 4) / 2, (0.5 + 1) / 2 on every rank
