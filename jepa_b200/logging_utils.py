"""Logging helpers with the reference's API (src/utils/logging.py).

`grad_logger` / `adamw_logger` return the same statistics as the reference but gather them with one
device->host transfer instead of one `float()` sync per tensor (~1000 syncs/step in the reference,
SURVEY.md section 5).
"""
import logging
import sys

import torch

LOG_FORMAT = "[%(levelname)-8s][%(asctime)s][%(funcName)-25s] %(message)s"
DATE_FORMAT = "%Y-%m-%d %H:%M:%S"


def gpu_timer(closure, log_timings=True):
    """Run closure(); return (result, elapsed GPU ms measured with CUDA events, -1 without CUDA)."""
    timed = log_timings and torch.cuda.is_available()
    if timed:
        t0 = torch.cuda.Event(enable_timing=True)
        t1 = torch.cuda.Event(enable_timing=True)
        t0.record()
    result = closure()
    elapsed = -1.
    if timed:
        t1.record()
        torch.cuda.synchronize()
        elapsed = t0.elapsed_time(t1)
    return result, elapsed


def get_logger(name=None, force=False):
    logging.basicConfig(stream=sys.stdout, level=logging.INFO, format=LOG_FORMAT, datefmt=DATE_FORMAT, force=force)
    return logging.getLogger(name=name)


class CSVLogger(object):
    """Append-mode CSV writer: header from (fmt, name) pairs, then one formatted row per log()."""

    def __init__(self, fname, *argv):
        self.fname = fname
        self.types = [fmt for fmt, _ in argv]
        with open(self.fname, '+a') as f:
            print(','.join(name for _, name in argv), file=f)

    def log(self, *argv):
        with open(self.fname, '+a') as f:
            print(','.join(fmt % v for fmt, v in zip(self.types, argv)), file=f)


class AverageMeter(object):
    """Running value / sum / count / avg / min / max."""

    def __init__(self):
        self.reset()

    def reset(self):
        self.val = 0
        self.avg = 0
        self.max = float('-inf')
        self.min = float('inf')
        self.sum = 0
        self.count = 0

    def update(self, val, n=1):
        self.val = val
        try:
            self.max = max(val, self.max)
            self.min = min(val, self.min)
        except Exception:
            pass
        self.sum += val * n
        self.count += n
        self.avg = self.sum / self.count


def _to_floats(tensors):
    if not tensors:
        return []
    return torch.stack([t.float().reshape(()) for t in tensors]).tolist()


def _flat_grad_sumsq(params):
    """(store, gradient buffer, per-tensor sums of squares, rows) when every parameter of `params` (all with a .grad) is
    a trainable member of ONE FlatParamStore and the gradients are slices of its flat buffer, else None.  params[i]'s
    sum of squares is sumsq[rows[i]]; the sums are those the unscale pass of this step left when still current."""
    store = getattr(params[0], "_vj_store", None)
    if store is None or not all(getattr(p, "_vj_store", None) is store and store.owns(p) for p in params):
        return None
    gflat = store.grad_buffer(params)
    if gflat is None:
        return None
    index = {n: i for i, n in enumerate(store.segments()[1])}
    if not all(p._vj_name in index for p in params):
        return None
    return store, gflat, store.grad_sumsq(gflat), [index[p._vj_name] for p in params]


def grad_logger(named_params):
    """Per-weight-tensor grad L2 norms: avg/min/max + first/last `qkv` layer (logging.py:91-105).  One segmented
    reduction over the flat gradient buffer (usually the one scaler.unscale_ already ran) and ONE device->host copy."""
    named = [(n, p) for n, p in named_params
             if (p.grad is not None) and not (n.endswith('.bias') or len(p.shape) == 1)]
    names = [n for n, _ in named]
    norms = []
    if named:
        flat = _flat_grad_sumsq([p for _, p in named]) if named[0][1].is_cuda else None
        if flat is not None:
            _, _, sumsq, rows = flat
            host = sumsq.sqrt().tolist()                      # the only host sync
            norms = [host[i] for i in rows]
        else:
            norms = _to_floats(list(torch._foreach_norm([p.grad.data for _, p in named])))
    stats = AverageMeter()
    stats.first_layer = None
    stats.last_layer = None
    for n, g in zip(names, norms):
        stats.update(g)
        if 'qkv' in n:
            stats.last_layer = g
            if stats.first_layer is None:
                stats.first_layer = g
    if stats.first_layer is None or stats.last_layer is None:
        stats.first_layer = stats.last_layer = 0.
    return stats


def adamw_logger(optimizer):
    """Mean |exp_avg| and |exp_avg_sq| per state tensor -> AverageMeters (logging.py:108-118).  FlatAdamW keeps both
    moments of a backbone in one flat buffer each: two segmented |x| reductions per backbone, one device->host copy."""
    from . import kernels as K
    from .optim import FlatAdamW
    vals1, vals2 = [], []
    covered = set()
    if isinstance(optimizer, FlatAdamW):
        parts = []
        for store, m, v, params in optimizer.flat_moments():
            seg, names = store.segments()
            out = torch.zeros(2, len(names), dtype=torch.float32, device=store.flat.device)
            K.seg_abs_sum(m, seg, out[0])
            K.seg_abs_sum(v, seg, out[1])
            numel = torch.tensor([store.offsets[n][1] for n in names], dtype=torch.float32)
            parts.append((out, numel))
            covered |= params
        for out, numel in parts:
            host = out.cpu()                                  # one copy per backbone
            vals1 += (host[0] / numel).tolist()
            vals2 += (host[1] / numel).tolist()
    rest = [s for p, s in optimizer.state.items() if p not in covered and s.get('exp_avg') is not None]
    if rest:
        vals1 += _to_floats([s.get('exp_avg').abs().mean() for s in rest])
        vals2 += _to_floats([s.get('exp_avg_sq').abs().mean() for s in rest])
    exp_avg_stats, exp_avg_sq_stats = AverageMeter(), AverageMeter()
    for a, b in zip(vals1, vals2):
        exp_avg_stats.update(a)
        exp_avg_sq_stats.update(b)
    return {'exp_avg': exp_avg_stats, 'exp_avg_sq': exp_avg_sq_stats}
