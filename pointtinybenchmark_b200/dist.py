"""Multi-GPU plumbing of the head (SURVEY.md §8e): images are the independent units, every rank runs the whole head on its own
images, inference needs no collective at all.  Training has exactly one exchange step — the gradient all-reduce the reference gets
from MMDistributedDataParallel (mmdet/apis/train.py:75-86) — done here for the head's parameters as ONE flat fp32 bucket over
NCCL (9.6 MB for the shipped head: a single NVLink/NVSwitch all-reduce, latency-bound, so no bucketing by layer).  The loss
normalisers stay rank-local like the reference's (cpr_head.py:1180, 1227; no reduce_mean)."""
import torch
import torch.distributed as dist


def reduce_mean_(tensor, group=None):
    """reduce_mean (mmdet core/utils/dist_utils.py:63-69) of a device tensor, in place: divided by the world size, then summed over the
    ranks in one all-reduce.  Unchanged when torch.distributed is not initialised.  The FCOS loss averages its two normalisers (positive
    count, centerness sum) this way as one two-element tensor, without a host synchronisation."""
    if not (dist.is_available() and dist.is_initialized()):
        return tensor
    tensor.div_(dist.get_world_size(group))
    dist.all_reduce(tensor, op=dist.ReduceOp.SUM, group=group)
    return tensor


def allreduce_grads(module, group=None, average=True):
    """all-reduce (sum, then / world) the gradients of `module`'s parameters in place through one flat bucket.
    Parameters without a gradient on this rank contribute zeros (DDP's find_unused_parameters semantics).  Returns the number
    of bytes exchanged per rank (0 when not distributed)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return 0
    params = [p for p in module.parameters() if p.requires_grad]
    if not params:
        return 0
    dev, dt = params[0].device, torch.float32
    sizes = [p.numel() for p in params]
    flat = torch.zeros(sum(sizes), dtype=dt, device=dev)
    o = 0
    for p, n in zip(params, sizes):
        if p.grad is not None:
            flat[o:o + n].copy_(p.grad.reshape(-1))
        o += n
    dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
    if average:
        flat.div_(dist.get_world_size(group))
    o = 0
    for p, n in zip(params, sizes):
        g = flat[o:o + n].view_as(p)
        if p.grad is None:
            p.grad = g.clone()
        else:
            p.grad.copy_(g)
        o += n
    return flat.numel() * flat.element_size()


class GradBucket:
    """The head's gradient exchange, overlapped with backward (VERDICT r1 item 5; reference: MMDistributedDataParallel's bucketed
    all-reduce, mmdet/apis/train.py:75-86, core/utils/dist_utils.py:25-51).

    * every parameter's `.grad` is a VIEW into ONE persistent flat fp32 buffer (autograd accumulates in place), so there is no
      copy-in / copy-out and no per-step allocation: `zero()` is one memset;
    * the parameters are grouped into buckets in the order their gradients become ready during backward (the loss-side classifiers
      first, then the tower layers last to first); a post-accumulate hook counts a bucket's parameters and, when the last one has
      landed, launches that bucket's all-reduce on a side stream behind an event — it runs under the remaining backward kernels; only
      the first tower layer's bucket (2.4 MB of the 9.6 MB) is exposed at the end of the step;
    * the mean over ranks is NCCL's own pre-multiplied sum (ReduceOp.AVG), no extra division kernel (gloo: sum, then one div_).
    Usage per step:  bucket.zero(); loss.backward(); bucket.wait()  [then the optimizer reads p.grad as usual].
    The bucketed / hooked exchange is opt-in (overlap=True); the default is one all-reduce of the flat buffer (see __init__)."""

    def __init__(self, module, group=None, average=True, buckets=None, overlap=False):
        # overlap=False (default): ONE all-reduce of the whole flat buffer (the head's 9.6 MB), issued by wait(): on an NVLink-connected
        # node that exchange is short, and per-bucket hooks add host work to a backward pass that is partly launch-bound.  overlap=True:
        # per-bucket all-reduces from post-accumulate hooks on a side stream, for heads / links where the exchange is long enough to be
        # worth hiding.
        self.group, self.average, self.overlap = group, average, overlap
        params = [(n, p) for n, p in module.named_parameters() if p.requires_grad]
        if buckets is None:
            buckets = self._default_buckets(params)
        order = [p for b in buckets for p in b]
        assert len(order) == len(params) and len({id(p) for p in order}) == len(order)
        self.flat = torch.zeros(sum(p.numel() for p in order), dtype=torch.float32, device=order[0].device)
        self.ranges, self._bucket_of, o = [], {}, 0
        for bi, b in enumerate(buckets):
            start = o
            for p in b:
                p.grad = self.flat[o:o + p.numel()].view_as(p)
                self._bucket_of[id(p)] = bi
                o += p.numel()
            self.ranges.append((start, o))
        self._need = [len(b) for b in buckets]
        self._left = list(self._need)
        self._next = 0            # collectives must be issued in the SAME order on every rank: strictly by bucket index
        self._works = []
        self._handles = [p.register_post_accumulate_grad_hook(self._hook) for p in order] if overlap else []
        self.world = dist.get_world_size(group) if (dist.is_available() and dist.is_initialized()) else 1
        self.comm_stream = torch.cuda.Stream(device=self.flat.device) if (self.flat.is_cuda and self.world > 1) else None
        self.nbytes = self.flat.numel() * 4

    @staticmethod
    def _default_buckets(named):
        """readiness order of the CPR / P2P heads: everything that is not a tower ConvModule first (classifiers: their gradients come
        out of the loss function), then `*_convs.{i}` from the last layer to the first."""
        import re
        layers, rest = {}, []
        for n, p in named:
            m = re.match(r'(\w+_convs)\.(\d+)\.', n)
            if m:
                layers.setdefault((int(m.group(2)), m.group(1)), []).append(p)
            else:
                rest.append(p)
        out = [rest] if rest else []
        for key in sorted(layers, key=lambda k: (-k[0], k[1])):
            out.append(layers[key])
        return out

    def zero(self):
        self.flat.zero_()
        self._left = list(self._need)
        self._next = 0
        self._works = []

    def _launch(self, bi):
        if self.world == 1:
            return
        a, b = self.ranges[bi]
        view = self.flat[a:b]
        nccl = dist.get_backend(self.group) == 'nccl'
        op = dist.ReduceOp.AVG if (self.average and nccl) else dist.ReduceOp.SUM
        if self.comm_stream is not None:
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(self.flat.device))
            with torch.cuda.stream(self.comm_stream):
                self.comm_stream.wait_event(ev)                    # the bucket's last gradient kernel has finished
                w = dist.all_reduce(view, op=op, group=self.group, async_op=True)
        else:
            w = dist.all_reduce(view, op=op, group=self.group, async_op=True)
        self._works.append((w, view, self.average and not nccl))

    def _hook(self, p):
        bi = self._bucket_of[id(p)]
        self._left[bi] -= 1
        while self._next < len(self._left) and self._left[self._next] == 0:      # in index order only (a bucket with a parameter that
            self._launch(self._next)                                            # is unused on this rank waits for wait())
            self._next += 1

    def wait(self):
        """the current stream waits for every bucket's all-reduce; buckets whose hooks never fired (parameters unused this step: their
        slice is still zero) are exchanged now, so every rank issues the same collectives."""
        if not self.overlap:
            if self.world > 1:
                nccl = dist.get_backend(self.group) == 'nccl'
                dist.all_reduce(self.flat, op=dist.ReduceOp.AVG if (self.average and nccl) else dist.ReduceOp.SUM, group=self.group)
                if self.average and not nccl:
                    self.flat.div_(self.world)
            return self.nbytes if self.world > 1 else 0
        while self._next < len(self._left):
            self._launch(self._next)
            self._next += 1
        for w, view, div in self._works:
            w.wait()
            if div:
                view.div_(self.world)
        self._works = []
        return self.nbytes if self.world > 1 else 0

    def close(self):
        for h in self._handles:
            h.remove()


def parse_losses(losses, group=None):
    """BaseDetector._parse_losses (mmdet/models/detectors/base.py:179-212): mean every entry (lists are summed), total `loss` = the sum
    of the entries whose key contains 'loss', and the logged values averaged over the ranks.  The reference issues one all-reduce and
    one `.item()` host sync PER scalar (4-6 per iteration); here the scalars travel as ONE packed tensor and come back with one copy.
    returns (loss tensor for backward — rank-local, like the reference —, {name: float})."""
    from collections import OrderedDict
    log_vars = OrderedDict()
    for k, v in losses.items():
        if isinstance(v, torch.Tensor):
            log_vars[k] = v.mean()
        elif isinstance(v, list):
            log_vars[k] = sum(x.mean() for x in v)
        else:
            raise TypeError(f'{k} is not a tensor or list of tensors')
    loss = sum(v for k, v in log_vars.items() if 'loss' in k)
    log_vars['loss'] = loss
    packed = torch.stack([v.detach().float().reshape(()) for v in log_vars.values()])
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        packed = packed / dist.get_world_size(group)
        dist.all_reduce(packed, op=dist.ReduceOp.SUM, group=group)
    vals = packed.cpu().tolist()
    return loss, OrderedDict(zip(log_vars.keys(), vals))
