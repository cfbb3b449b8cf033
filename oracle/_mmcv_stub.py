"""Test scaffolding ONLY (not product code, not shipped on any product path).

Auto-stubs the un-vendored third-party packages (`mmcv`, `pycocotools`, `matplotlib`, ...)
so that the *real, unmodified* reference package at /root/reference/TOV_mmdetection/mmdet can be
imported on CPU in the build container.  Used by `oracle/make_golden.py` to pin the oracle
restatement against the reference itself and to generate `tests/golden/*`.

/root/reference does not exist on the GPU box, so nothing under tests/ -m gpu, smoke() or
bench.py imports this file.

Third-party arithmetic restated here (no source under /root/reference):
  * mmcv.ops.nms / batched_nms  (mmcv-full 1.3.x): class-offset trick + greedy IoU>thr NMS,
    pinned to torchvision.ops.nms on CPU (same IoU > thr, offset 0 rule).
  * mmcv.ops.sigmoid_focal_loss: formula restated in-tree by the reference as
    py_sigmoid_focal_loss (mmdet/models/losses/focal_loss.py:11-56); mapped to that.
  * mmcv.cnn.ConvModule: conv(bias iff no norm) + GN/BN + ReLU with mmcv's submodule names
    (`conv`, `gn`/`bn`, `activate`).
"""
import sys, types, importlib.abc, importlib.machinery
import torch, torch.nn as nn
import torch.nn.functional as F

REFERENCE_ROOT = '/root/reference/TOV_mmdetection'


class Registry:
    def __init__(self, name, parent=None, build_func=None, scope=None):
        self.name = name
        self.module_dict = {}
        self.parent = parent

    def get(self, key):
        if key in self.module_dict:
            return self.module_dict[key]
        return self.parent.get(key) if self.parent is not None else None

    def register_module(self, name=None, force=False, module=None):
        if module is not None:
            self.module_dict[name or module.__name__] = module
            return module

        def deco(cls):
            names = [name] if isinstance(name, str) else (name or [cls.__name__])
            for n in names:
                self.module_dict[n] = cls
            return cls
        return deco

    def build(self, cfg, default_args=None):
        return build_from_cfg(cfg, self, default_args)


def build_from_cfg(cfg, registry, default_args=None):
    args = dict(cfg)
    if default_args:
        for k, v in default_args.items():
            args.setdefault(k, v)
    t = args.pop('type')
    cls = registry.get(t) if isinstance(t, str) else t
    if cls is None:
        raise KeyError(f'{t} not in {registry.name}')
    return cls(**args)


class BaseModule(nn.Module):
    def __init__(self, init_cfg=None):
        super().__init__()
        self.init_cfg = init_cfg

    def init_weights(self):
        pass


class ConvModule(nn.Module):
    def __init__(self, cin, cout, k, stride=1, padding=0, dilation=1, groups=1, bias='auto',
                 conv_cfg=None, norm_cfg=None, act_cfg=dict(type='ReLU'), inplace=True, **kw):
        super().__init__()
        wn = norm_cfg is not None
        if bias == 'auto':
            bias = not wn
        self.conv = nn.Conv2d(cin, cout, k, stride, padding, dilation, groups, bias=bias)
        self.norm_name = None
        if wn:
            if norm_cfg['type'] == 'GN':
                self.norm_name = 'gn'
                self.add_module('gn', nn.GroupNorm(norm_cfg['num_groups'], cout))
            else:
                self.norm_name = 'bn'
                self.add_module('bn', nn.BatchNorm2d(cout))
        self.activate = nn.ReLU(inplace=inplace) if act_cfg else None

    def forward(self, x):
        x = self.conv(x)
        if self.norm_name is not None:
            x = getattr(self, self.norm_name)(x)
        return self.activate(x) if self.activate is not None else x


def _deco_factory(*a, **k):
    if len(a) == 1 and callable(a[0]) and not k:
        return a[0]
    return lambda f: f


def nms(boxes, scores, iou_threshold, offset=0, score_threshold=0, max_num=-1):
    import torchvision
    assert offset == 0
    keep = torchvision.ops.nms(boxes, scores, float(iou_threshold))
    if max_num > 0:
        keep = keep[:max_num]
    return torch.cat([boxes[keep], scores[keep, None]], 1), keep


def batched_nms(boxes, scores, idxs, nms_cfg, class_agnostic=False):
    cfg = dict(nms_cfg)
    class_agnostic = cfg.pop('class_agnostic', class_agnostic)
    if class_agnostic:
        b = boxes
    else:
        b = boxes + (idxs.to(boxes) * (boxes.max() + 1))[:, None]
    t = cfg.pop('type', 'nms')
    assert t == 'nms'
    split_thr = cfg.pop('split_thr', 10000)
    if len(b) < split_thr:
        dets, keep = nms(b, scores, **cfg)
        return torch.cat([boxes[keep], dets[:, -1:]], -1), keep
    # mmcv 1.3.x at split_thr boxes or more: NMS class by class (by idxs, also when class_agnostic), kept entries sorted by
    # score (restated, unpinned)
    total = torch.zeros(scores.shape, dtype=torch.bool)
    for c in torch.unique(idxs):
        m = (idxs == c).nonzero(as_tuple=False).view(-1)
        total[m[nms(b[m], scores[m], **cfg)[1]]] = True
    keep = total.nonzero(as_tuple=False).view(-1)
    sc, inds = scores[keep].sort(descending=True, stable=True)
    keep = keep[inds]
    return torch.cat([boxes[keep], sc[:, None]], -1), keep


def sigmoid_focal_loss(pred, target, gamma=2.0, alpha=0.25, weight=None, reduction='none'):
    """mmcv op signature (pred, target(int64), gamma, alpha, None, 'none'); formula =
    reference py_sigmoid_focal_loss (losses/focal_loss.py:11-56) before weighting."""
    num_classes = pred.size(1)
    t = F.one_hot(target, num_classes=num_classes + 1)[:, :num_classes].type_as(pred)
    p = pred.sigmoid()
    pt = (1 - p) * t + p * (1 - t)
    fw = (alpha * t + (1 - alpha) * (1 - t)) * pt.pow(gamma)
    return F.binary_cross_entropy_with_logits(pred, t, reduction='none') * fw


KNOWN = {
    'mmcv': dict(__version__='1.3.8', jit=_deco_factory),
    'mmcv.utils': dict(Registry=Registry, build_from_cfg=build_from_cfg),
    'mmcv.cnn': dict(ConvModule=ConvModule, MODELS=Registry('model')),
    'mmcv.runner': dict(BaseModule=BaseModule, force_fp32=_deco_factory, auto_fp16=_deco_factory,
                        HOOKS=Registry('hook'), Hook=object, OptimizerHook=object),
    'mmcv.ops': dict(batched_nms=batched_nms, nms=nms, sigmoid_focal_loss=sigmoid_focal_loss),
    'mmcv.ops.nms': dict(batched_nms=batched_nms, nms=nms),
}
_REG_NAMES = ('MODELS', 'HOOKS', 'PIPELINES', 'DATASETS', 'ATTENTION', 'TRANSFORMER', 'RUNNERS', 'OPTIMIZERS')
_PREFIXES = ('mmcv', 'huicv', 'pycocotools', 'terminaltables', 'matplotlib', 'skimage',
             'cityscapesscripts', 'lvis', 'albumentations', 'imagecorruptions')


class _AutoModule(types.ModuleType):
    def __getattr__(self, n):
        if n.startswith('__'):
            raise AttributeError(n)
        if n.isupper() and ('_' in n or n in _REG_NAMES):
            v = Registry(n)
        elif n[:1].isupper():
            v = type(n, (nn.Module,), {'__init__': lambda s, *a, **k: nn.Module.__init__(s)})
        else:
            v = _deco_factory
        setattr(self, n, v)
        return v


class _Finder(importlib.abc.MetaPathFinder, importlib.abc.Loader):
    def find_spec(self, name, path, target=None):
        root = name.split('.')[0]
        if root in _PREFIXES:
            return importlib.machinery.ModuleSpec(name, self, is_package=True)

    def create_module(self, spec):
        m = _AutoModule(spec.name)
        m.__path__ = []
        m.__dict__.update(KNOWN.get(spec.name, {}))
        return m

    def exec_module(self, m):
        pass


class CfgDict(dict):
    """stand-in for mmcv.Config nodes: attribute access on dict."""
    __getattr__ = dict.get


_installed = False


def install():
    global _installed
    if _installed:
        return
    import os
    if not os.path.isdir(REFERENCE_ROOT):
        raise RuntimeError(f'{REFERENCE_ROOT} not present: the reference can only be imported in the build container')
    sys.meta_path.insert(0, _Finder())
    sys.path.insert(0, REFERENCE_ROOT)
    _installed = True


def load_reference():
    """returns the reference's HEADS registry (real mmdet code, stubbed mmcv)."""
    install()
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        import mmdet.models  # noqa
        from mmdet.models.builder import HEADS
    return HEADS
