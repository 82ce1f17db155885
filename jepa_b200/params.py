"""Flat parameter store: fp32 master weights of one backbone in ONE contiguous HBM buffer.

The reference keeps ~300 separate fp32 tensors per network and touches them one by one (autocast
weight casts, the EMA python loop at app/vjepa/train.py:484-487, foreach AdamW).  Here the
nn.Parameters of a backbone are re-pointed (``p.data``) into slices of a single buffer so that
  * the bf16 shadow the wgmma GEMMs read is produced by one cast launch per step,
  * the target-encoder EMA is one launch,
  * weight gradients are written by the wgrad GEMMs straight into one flat fp32 gradient buffer
    (one NCCL all-reduce region for data parallel).
Parameter identity, names, shapes and state_dict keys are untouched (drop-in contract,
SURVEY.md section 8b); ``copy.deepcopy`` / ``.to()`` / DDP broadcast keep working because the
store re-adopts the parameters lazily whenever they no longer alias its buffer.
"""
import torch

from . import kernels as K

ALIGN = 64  # elements; keeps every slice 256-byte aligned (TMA needs 16 B)


def padded_head_dim(hd):
    if hd <= 32:
        return 32
    if hd <= 64:
        return 64
    if hd <= 128:
        return 128
    raise ValueError(f"head dim {hd} > 128 is not supported by the attention kernels")


class FlatParamStore:
    def __init__(self):
        self.flat = None      # fp32 [total]
        self.shadow = None    # bf16 [total]
        self.offsets = {}     # name -> (offset, numel, shape)
        self.total = 0
        self._params = None
        self._shadow_fresh = False   # set by the kernels that emit the bf16 shadow together with a parameter update
        self._shadow_complete = False   # a full cast has filled every element of the shadow at least once
        self._seg = None             # uint16 per 64-element block -> index into named parameters (0xFFFF: frozen / padding)

    def __deepcopy__(self, memo):
        return FlatParamStore()  # copies re-adopt their own (deep-copied) parameters lazily

    # -- adoption ----------------------------------------------------------------------------
    def _aliases(self, named):
        if self.flat is None or self._params is None or len(named) != len(self._params):
            return False
        base = self.flat.data_ptr()
        for (name, p), (pname, q) in zip(named, self._params):
            if p is not q or name != pname:
                return False
            off, n, shape = self.offsets[name]
            if p.data_ptr() != base + 4 * off or tuple(p.shape) != shape or p.dtype != torch.float32:
                return False
        return True

    def adopt(self, module):
        """Make every parameter of `module` a view into the flat buffer (no-op if already so)."""
        named = [(n, p) for n, p in module.named_parameters()]
        if self._aliases(named):
            return self
        dev = named[0][1].device
        if dev.type != "cuda":
            raise RuntimeError("jepa_b200: parameters must be on a CUDA device (no CPU fallback for the hot path)")
        off = 0
        offsets = {}
        for n, p in named:
            offsets[n] = (off, p.numel(), tuple(p.shape))
            off += (p.numel() + ALIGN - 1) // ALIGN * ALIGN
        flat = torch.zeros(off, dtype=torch.float32, device=dev)
        with torch.no_grad():
            for n, p in named:
                o, cnt, shape = offsets[n]
                view = flat[o:o + cnt].view(shape)
                view.copy_(p.data.to(torch.float32))
                p.data = view
                p._vj_store, p._vj_name = self, n
        self.flat, self.offsets, self.total, self._params = flat, offsets, off, named
        self.shadow = torch.empty(off, dtype=torch.bfloat16, device=dev)
        self._shadow_fresh = False
        self._shadow_complete = False
        self._seg = None
        return self

    def owns(self, p):
        """True if parameter `p` currently aliases its slice of this store's flat buffer."""
        name = getattr(p, "_vj_name", None)
        if self.flat is None or name not in self.offsets:
            return False
        off, n, shape = self.offsets[name]
        return p.data_ptr() == self.flat.data_ptr() + 4 * off and tuple(p.shape) == shape

    # -- per-step products ---------------------------------------------------------------------
    def refresh_shadow(self):
        """bf16 operands of this forward.  The fused AdamW / EMA kernels already wrote them together with the parameter
        update (one pass instead of update + cast); that copy is valid for exactly one refresh, anything else that may
        have touched the parameters in between (load_state_dict, manual edits) is covered by casting again."""
        if self._shadow_fresh:
            self._shadow_fresh = False
            return
        K.cast_f32_bf16(self.flat, self.shadow)
        self._shadow_complete = True

    def mark_shadow_fresh(self, complete=False):
        # AdamW only writes the elements it updates (frozen tensors and alignment padding are skipped), so its copy is
        # complete only on top of a shadow a full pass (cast, or the EMA kernel: complete=True) has filled at least once
        if complete:
            self._shadow_complete = True
        self._shadow_fresh = self._shadow_complete

    def invalidate_shadow(self):
        self._shadow_fresh = False

    def segments(self):
        """(seg uint16 [total/64] on the device, names): block -> index of the TRAINABLE tensor it belongs to."""
        if self._seg is None:
            seg = torch.full((self.total // ALIGN,), 0xFFFF, dtype=torch.int32)
            names = []
            for n, p in self._params:
                if not p.requires_grad:
                    continue
                off, cnt, _ = self.offsets[n]
                seg[off // ALIGN:(off + cnt + ALIGN - 1) // ALIGN] = len(names)
                names.append(n)
            self._seg = (seg.to(torch.uint16).to(self.flat.device), names)
        return self._seg

    def bf16(self, name):
        o, n, shape = self.offsets[name]
        return self.shadow[o:o + n].view(shape)

    def f32(self, name):
        o, n, shape = self.offsets[name]
        return self.flat[o:o + n].view(shape)

    def new_grad_buffer(self):
        self._grad_gen = getattr(self, "_grad_gen", 0) + 1     # invalidates cached per-tensor gradient statistics
        return torch.zeros(self.total, dtype=torch.float32, device=self.flat.device)

    def grad_view(self, gflat, name):
        o, n, shape = self.offsets[name]
        return gflat[o:o + n].view(shape)
