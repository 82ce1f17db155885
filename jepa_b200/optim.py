"""AdamW on our own kernels with torch.optim.Optimizer's interface.

Drop-in for the `torch.optim.AdamW(param_groups, betas, eps)` the reference builds in
app/vjepa/utils.py:173-194: same param_groups / state layout (`step`, `exp_avg`, `exp_avg_sq`), so the
LR / WD schedulers, `adamw_logger`, `state_dict()` and reference checkpoints all keep working.
`_step_supports_amp_scaling` makes torch's GradScaler hand over `found_inf` / `grad_scale` as device
tensors instead of syncing the host: the skip-on-overflow decision is taken inside the kernel.

Fast path: when all parameters of a backbone live in a FlatParamStore and their gradients are the slices
of ONE flat gradient buffer (what our backward produces), the whole backbone is updated by a single
`vj_adamw_flat` launch; a per-64-element group table carries each tensor's (lr, weight_decay) group.
Anything else falls back to one `vj_adamw_step` launch per tensor.  A trainable member of a store whose `.grad` is None
(the attentive probe's `proj`, which the reference never applies) is treated as torch.optim.AdamW treats it: it is not
updated and gets no optimizer state.
"""
import ctypes

import torch

from . import _lib
from . import kernels as K


class FlatGradScaler(torch.cuda.amp.GradScaler):
    """torch's GradScaler (same state_dict, same scale / growth policy, app/vjepa/utils.py:209) whose unscale pass over
    FlatAdamW-owned flat gradient buffers is one of our kernels instead of torch._amp_foreach_non_finite_check_and_unscale_
    over hundreds of views; anything not in a flat buffer still goes through torch's implementation."""

    def _unscale_grads_(self, optimizer, inv_scale, found_inf, allow_fp16):
        if not isinstance(optimizer, FlatAdamW):
            return super()._unscale_grads_(optimizer, inv_scale, found_inf, allow_fp16)
        inv = inv_scale.reshape(1).contiguous()
        fi = found_inf.reshape(1)
        rest = optimizer.unscale_flat_(inv, fi)
        if rest:
            grads = [p.grad for p in rest]
            torch._amp_foreach_non_finite_check_and_unscale_(grads, found_inf, inv_scale)
        return {found_inf.device: found_inf}


class FlatAdamW(torch.optim.Optimizer):
    _step_supports_amp_scaling = True

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2):
        if lr < 0 or eps < 0 or not (0 <= betas[0] < 1) or not (0 <= betas[1] < 1):
            raise ValueError("invalid AdamW hyper-parameters")
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        self._flat = {}   # id(store) -> dict(store, gid, m, v, step, key)

    # ------------------------------------------------------------------------------------------ flat path
    def _flat_plan(self):
        """Group parameters by FlatParamStore; returns (plans, leftovers)."""
        by_store, leftovers = {}, []
        for gi, group in enumerate(self.param_groups):
            for p in group['params']:
                store = getattr(p, "_vj_store", None)
                if store is None or gi > 3 or not store.owns(p):
                    leftovers.append((gi, p))
                else:
                    by_store.setdefault(id(store), (store, []))[1].append((gi, p))
        return by_store, leftovers

    @staticmethod
    def _stepped(p):
        """Members the flat step updates: trainable and with a gradient this step (torch.optim.AdamW skips the rest)."""
        return p.requires_grad and p.grad is not None

    def _flat_state(self, store, members):
        key = (store.flat.data_ptr(), store.total, tuple((gi, id(p), self._stepped(p)) for gi, p in members))
        st = self._flat.get(id(store))
        if st is not None and st["key"] == key:
            p0 = next(p for _, p in members if self._stepped(p))   # frozen / gradient-less members carry no state
            off0 = store.offsets[p0._vj_name][0]
            ea = self.state.get(p0, {}).get("exp_avg")
            if ea is not None and ea.data_ptr() == st["m"].data_ptr() + 4 * off0:
                return st          # state still aliases the flat moment buffers (not replaced by load_state_dict)
        dev = store.flat.device
        gid = torch.full((store.total // 64,), 255, dtype=torch.uint8)
        for gi, p in members:
            off, n, _ = store.offsets[p._vj_name]
            gid[off // 64:(off + n + 63) // 64] = gi if self._stepped(p) else 255   # frozen (pos_embed): untouched
        m = torch.zeros(store.total, dtype=torch.float32, device=dev)
        v = torch.zeros(store.total, dtype=torch.float32, device=dev)
        # the step count is a DEVICE scalar (as in torch's fused / capturable AdamW): the kernel advances it only when the
        # GradScaler did not skip the step, so bias correction and the checkpointed `step` do not drift on overflow skips
        step = torch.zeros((), dtype=torch.float32, device=dev)
        for _, p in members:       # resume: carry per-tensor state (e.g. from load_state_dict) into the flat buffers
            old = self.state.get(p, {})
            if "step" in old:
                step.fill_(float(old["step"]))
                break
        for gi, p in members:
            if not self._stepped(p):    # torch.optim.AdamW never creates state for a parameter without a gradient (the frozen
                continue                # pos_embed, the probe's proj): keep state_dict() entry-for-entry identical
            off, n, shape = store.offsets[p._vj_name]
            old = self.state.get(p, {})
            if "exp_avg" in old:
                m[off:off + n].view(shape).copy_(old["exp_avg"])
                v[off:off + n].view(shape).copy_(old["exp_avg_sq"])
            self.state[p] = {"step": step, "exp_avg": m[off:off + n].view(shape), "exp_avg_sq": v[off:off + n].view(shape)}
        st = dict(store=store, gid=gid.to(dev), m=m, v=v, step=step, key=key)
        self._flat[id(store)] = st
        return st

    @staticmethod
    def _flat_grad_base(store, members):
        """Device pointer of the flat gradient buffer if every member's .grad is its slice of one buffer.  Members without
        a gradient are skipped (not stepped, see _stepped)."""
        base = None
        for _, p in members:
            g = p.grad
            if g is None:
                continue
            if g.dtype != torch.float32 or not g.is_contiguous():
                return None
            off = store.offsets[p._vj_name][0]
            b = g.data_ptr() - 4 * off
            if base is None:
                base = b
            elif b != base:
                return None
        return base

    # ------------------------------------------------------------------------------------------ GradScaler hook
    @torch.no_grad()
    def unscale_flat_(self, inv_scale, found_inf):
        """scaler.unscale_ for gradients that live in flat buffers: ONE kernel per backbone unscales in place, raises the
        non-finite flag and leaves per-tensor sums of squares behind for grad_logger / clip_grad_norm_ (no host sync).
        Returns the parameters it did not cover (torch's foreach path handles those)."""
        by_store, leftovers = self._flat_plan()
        self._grad_stats = {}
        for store, members in by_store.values():
            base = self._flat_grad_base(store, members)
            if base is None:
                leftovers.extend(members)
                continue
            seg, names = store.segments()
            sumsq = torch.zeros(len(names), dtype=torch.float32, device=store.flat.device)
            _lib.call("vj_grad_unscale_stats", base, seg.data_ptr(), store.total, K._p(inv_scale), K._p(found_inf),
                      sumsq.data_ptr(), 1, K._s())
            self._grad_stats[id(store)] = (store, base, sumsq, names)
            store._grad_sumsq = (base, getattr(store, "_grad_gen", 0), sumsq)   # reused by grad_logger / clip_grad_norm_
        return [p for _, p in leftovers if p.grad is not None]

    def grad_stats_for(self, store):
        """(sumsq tensor, names) left by the last unscale_flat_ for this store, or None."""
        hit = getattr(self, "_grad_stats", {}).get(id(store))
        return None if hit is None else (hit[2], hit[3])

    def zero_grad(self, set_to_none=True):
        self._grad_stats = {}
        return super().zero_grad(set_to_none=set_to_none)

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        found_inf = getattr(self, "found_inf", None)
        grad_scale = getattr(self, "grad_scale", None)
        inv_scale = None
        if grad_scale is not None:
            inv_scale = grad_scale.double().reciprocal().float().reshape(1).contiguous()
        if found_inf is not None:
            found_inf = found_inf.float().reshape(1).contiguous()

        by_store, leftovers = self._flat_plan()
        for store, members in by_store.values():
            base = self._flat_grad_base(store, members)
            # parameters of the store that are NOT optimised here (frozen ones) stay untouched: group id 255
            if base is None:
                leftovers.extend(members)
                continue
            st = self._flat_state(store, members)
            lr4 = (ctypes.c_float * 4)(*[float(g['lr']) for g in self.param_groups[:4]] + [0.0] * (4 - min(4, len(self.param_groups))))
            wd4 = (ctypes.c_float * 4)(*[float(g['weight_decay']) for g in self.param_groups[:4]] + [0.0] * (4 - min(4, len(self.param_groups))))
            beta1, beta2 = self.param_groups[0]['betas']
            _lib.call("vj_adamw_flat", store.flat.data_ptr(), base, st["m"].data_ptr(), st["v"].data_ptr(),
                      st["gid"].data_ptr(), store.total, ctypes.cast(lr4, ctypes.c_void_p), ctypes.cast(wd4, ctypes.c_void_p),
                      float(beta1), float(beta2), float(self.param_groups[0]['eps']), 0,
                      K._p(inv_scale), K._p(found_inf), st["step"].data_ptr(), store.shadow.data_ptr(), K._s())
            store.mark_shadow_fresh()     # the kernel wrote next step's bf16 operands with the update (if not skipped,
                                          # and if skipped the previous shadow is still the right one)

        for gi, p in leftovers:
            if p.grad is None:
                continue
            group = self.param_groups[gi]
            beta1, beta2 = group['betas']
            if not p.is_cuda:
                raise RuntimeError("FlatAdamW: parameters must be CUDA tensors (no CPU fallback)")
            state = self.state[p]
            if len(state) == 0:
                state['step'] = torch.zeros((), dtype=torch.float32)
                state['exp_avg'] = torch.zeros_like(p, memory_format=torch.preserve_format)
                state['exp_avg_sq'] = torch.zeros_like(p, memory_format=torch.preserve_format)
            state['step'] += 1
            g = p.grad
            if g.dtype != torch.float32 or not g.is_contiguous():
                g = g.float().contiguous()
            n = p.numel()
            if n % 4 != 0 or p.data_ptr() % 16 or g.data_ptr() % 16 or not p.is_contiguous():
                raise RuntimeError(f"FlatAdamW: parameter of {n} elements is not 16-byte vectorisable; "
                                   "adopt the module into a FlatParamStore first")
            K.adamw_step(p, g, state['exp_avg'], state['exp_avg_sq'], group['lr'], beta1, beta2, group['eps'],
                         group['weight_decay'], int(state['step']), inv_scale, found_inf)
        return loss
