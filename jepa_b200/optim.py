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
import torch

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

    def _in_flat_moments(self, st, name, p):
        """True if p's exp_avg is still its slice of the flat moment buffer of `st` (load_state_dict replaces it)."""
        ea = self.state.get(p, {}).get("exp_avg")
        return ea is not None and ea.data_ptr() == st["m"].data_ptr() + 4 * st["store"].offsets[name][0]

    def flat_moments(self):
        """[(store, m, v, params)]: the flat first / second moment buffers of each store stepped by one launch, and the
        parameters whose exp_avg / exp_avg_sq are still slices of them."""
        return [(st["store"], st["m"], st["v"], {p for n, p in st["store"]._params if self._in_flat_moments(st, n, p)})
                for st in self._flat.values()]

    def _flat_state(self, store, members):
        key = (store.flat.data_ptr(), store.total, tuple((gi, id(p), self._stepped(p)) for gi, p in members))
        st = self._flat.get(id(store))
        if st is not None and st["key"] == key:
            p0 = next(p for _, p in members if self._stepped(p))   # frozen / gradient-less members carry no state
            if self._in_flat_moments(st, p0._vj_name, p0):
                return st
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

    # ------------------------------------------------------------------------------------------ GradScaler hook
    @torch.no_grad()
    def unscale_flat_(self, inv_scale, found_inf):
        """scaler.unscale_ for gradients that live in flat buffers: ONE kernel per backbone unscales in place, raises the
        non-finite flag and leaves per-tensor sums of squares behind for grad_logger / clip_grad_norm_ (no host sync).
        Returns the parameters it did not cover (torch's foreach path handles those)."""
        by_store, leftovers = self._flat_plan()
        for store, members in by_store.values():
            gflat = store.grad_buffer(p for _, p in members)
            if gflat is None:
                leftovers.extend(members)
            else:
                store.grad_sumsq(gflat, inv_scale, found_inf)
        return [p for _, p in leftovers if p.grad is not None]

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
            gflat = store.grad_buffer(p for _, p in members)
            # parameters of the store that are NOT optimised here (frozen ones) stay untouched: group id 255
            if gflat is None:
                leftovers.extend(members)
                continue
            st = self._flat_state(store, members)
            groups = self.param_groups[:4]
            beta1, beta2 = self.param_groups[0]['betas']
            K.adamw_flat(store.flat, gflat, st["m"], st["v"], st["gid"], [g['lr'] for g in groups],
                         [g['weight_decay'] for g in groups], beta1, beta2, self.param_groups[0]['eps'], st["step"],
                         store.shadow, inv_scale, found_inf)
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
