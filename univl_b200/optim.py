"""Fused BertAdam over flat buffers + the flat gradient layout the layer kernels accumulate into directly.

`FusedBertAdam` reproduces the reference optimizer (modules/optimization.py:66-167: no bias correction, eps outside
the sqrt, decoupled weight decay, per-tensor gradient clipping, warmup_linear schedule with a per-step counter) and
the driver's global `clip_grad_norm_` (main_task_retrieval.py:347) in three kernel launches for the whole model
(csrc/optim.cu), instead of a Python loop of ~10 launches over ~300 tensors.

Flat layout: all parameters live in ONE fp32 buffer (`p.data` become views — `state_dict()` is unchanged), gradients
in a second one (`p.grad` are views).  Two-dimensional weights keep the offsets of the bf16 weight arena
(runtime.WeightArena: q/k/v adjacent), so the update kernel writes the bf16 copy the GEMMs consume in the same pass
and the arena needs no separate refresh; 1-D parameters follow.  With `sink_grads=True` the backward kernels
accumulate (red.global.add) straight into the flat gradient views — no per-parameter autograd accumulation — which is
also what the gradient all-reduce (univl_b200/ddp.py) operates on in place.
"""
import torch

from . import runtime as rt
from .runtime import call


def _align(n, a=64):
    return (n + a - 1) // a * a


def _zero(flat):
    """clear a flat fp32 buffer through the C ABI (cudaMemsetAsync on the current stream; capturable)"""
    call("univl_fill_f32", flat.data_ptr(), 0.0, flat.numel())


class FlatParams:
    """Flatten a model's parameters/gradients (idempotent per model)."""

    def __init__(self, model, device):
        arena = rt.arena_of(model)
        with torch.cuda.device(device):
            if arena.buf is None or arena.device != device:
                arena._build(device)
        self.model, self.arena, self.device = model, arena, device
        self.params, self.offsets = [], []
        seen = set()
        for p, off, n in arena.entries:          # 2-D weights at their arena offsets
            self.params.append(p)
            self.offsets.append(off)
            seen.add(id(p))
        total = arena.buf.numel()
        for p in model.parameters():             # 1-D (and any other) parameters afterwards
            if id(p) in seen:
                continue
            seen.add(id(p))
            self.params.append(p)
            self.offsets.append(total)
            total += _align(p.numel())
        self.total = total
        self.p = torch.zeros(total, dtype=torch.float32, device=device)
        self.g = torch.zeros(total, dtype=torch.float32, device=device)
        self.shadow = torch.zeros(total, dtype=torch.bfloat16, device=device)
        for p, off in zip(self.params, self.offsets):
            n = p.numel()
            self.p[off:off + n].copy_(p.data.reshape(-1))
            p.data = self.p[off:off + n].view(p.shape)
            p.grad = self.g[off:off + n].view(p.shape)
        # the arena now aliases the shadow buffer (same offsets) and is refreshed by the optimizer kernel
        call("univl_cast_f32_to_bf16", self.p.data_ptr(), self.shadow.data_ptr(), total)
        arena.buf = self.shadow
        arena._ptrs = None
        arena.fresh = True
        self.by_id = {id(p): (off, p.numel(), tuple(p.shape)) for p, off in zip(self.params, self.offsets)}
        # keyed by storage address: autograd may hand backward a different Python wrapper of the same parameter
        self.by_ptr = {p.data_ptr(): (off, p.numel(), tuple(p.shape)) for p, off in zip(self.params, self.offsets)}
        model.__dict__["_univl_flat"] = self

    def has(self, param):
        return param.data_ptr() in self.by_ptr

    def grad_view(self, param):
        off, n, shape = self.by_ptr[param.data_ptr()]
        return self.g[off:off + n].view(shape)

    def grad_view_packed(self, params):
        """one contiguous view over adjacent parameters (q/k/v weights or biases); None if not adjacent"""
        off0, n0, shape0 = self.by_ptr[params[0].data_ptr()]
        off = off0
        for p in params:
            o, n, _ = self.by_ptr[p.data_ptr()]
            if o != off:
                return None
            off += n
        rows = sum(self.by_ptr[p.data_ptr()][2][0] for p in params)
        return self.g[off0:off].view((rows,) + shape0[1:])

    def zero_grad(self):
        _zero(self.g)


def flatten(model, sink_grads=True):
    """Move `model`'s parameters/gradients into flat buffers; optionally register the gradient sinks."""
    dev = next(model.parameters()).device
    flat = model.__dict__.get("_univl_flat")
    if flat is None or flat.model is not model:   # (a replica's __dict__ copy carries the original's entry)
        flat = FlatParams(model, dev)
    rt.set_grad_sink(flat if sink_grads else None, model)
    return flat


class FusedBertAdam(torch.optim.Optimizer):
    """BertAdam (reference modules/optimization.py:66) with the whole step fused on the device.

    Accepts the reference's constructor arguments.  `global_clip_norm` > 0 additionally applies the driver-side
    `clip_grad_norm_(model.parameters(), global_clip_norm)`; `grad_scale` multiplies gradients first (1/world_size
    after a sum all-reduce).  If `model` is given its parameters are flattened (see FlatParams) and the bf16 weight
    arena is kept fresh by the update kernel; otherwise the optimizer builds private flat buffers on first step.
    """

    def __init__(self, params, lr=1e-4, warmup=-1, t_total=-1, schedule="warmup_linear", b1=0.9, b2=0.999, e=1e-6,
                 weight_decay=0.01, max_grad_norm=1.0, global_clip_norm=-1.0, grad_scale=1.0, model=None,
                 sink_grads=True):
        if lr < 0.0:
            raise ValueError("Invalid learning rate: {} - should be >= 0.0".format(lr))
        if schedule not in ("warmup_linear",):
            raise ValueError("univl_b200 FusedBertAdam implements schedule 'warmup_linear' only (got %r)" % schedule)
        if not 0.0 <= warmup < 1.0 and not warmup == -1:
            raise ValueError("Invalid warmup: {} - should be in [0.0, 1.0[ or -1".format(warmup))
        for name, b in (("b1", b1), ("b2", b2)):
            if not 0.0 <= b < 1.0:
                raise ValueError("Invalid {} parameter: {} - should be in [0.0, 1.0[".format(name, b))
        if not e >= 0.0:
            raise ValueError("Invalid epsilon value: {} - should be >= 0.0".format(e))
        defaults = dict(lr=lr, schedule=schedule, warmup=warmup, t_total=t_total, b1=b1, b2=b2, e=e,
                        weight_decay=weight_decay, max_grad_norm=max_grad_norm)
        super(FusedBertAdam, self).__init__(params, defaults)
        self.global_clip_norm = float(global_clip_norm)
        self.grad_scale = float(grad_scale)
        # bf16 gradients to read INSTEAD of the fp32 buffer (the summed payload of ddp.FlatGradReducer(compress="bf16"));
        # set by the data-parallel loop, None = read self.g
        self.grad_payload = None
        self.model = model
        self.sink_grads = sink_grads
        self._built = False

    # ------------------------------------------------------------------------------------------------------
    def _build(self):
        first = self.param_groups[0]["params"][0]
        dev = first.device
        if dev.type != "cuda":
            raise RuntimeError("FusedBertAdam needs CUDA parameters (sm_90a kernels only)")
        if self.model is not None:
            flat = flatten(self.model, self.sink_grads)
            self.flat = flat
            self.p, self.g, self.shadow = flat.p, flat.g, flat.shadow
            lookup = flat.by_id
        else:
            plist = []
            seen = set()
            for grp in self.param_groups:
                for p in grp["params"]:
                    if id(p) not in seen:
                        seen.add(id(p))
                        plist.append(p)
            offs, total = [], 0
            for p in plist:
                offs.append(total)
                total += _align(p.numel())
            self.p = torch.zeros(total, dtype=torch.float32, device=dev)
            self.g = torch.zeros(total, dtype=torch.float32, device=dev)
            self.shadow = None
            for p, off in zip(plist, offs):
                n = p.numel()
                self.p[off:off + n].copy_(p.data.reshape(-1))
                p.data = self.p[off:off + n].view(p.shape)
            lookup = {id(p): (off, p.numel(), tuple(p.shape)) for p, off in zip(plist, offs)}
            self.flat = None
            self._plist, self._offs = plist, offs
        self.m = torch.zeros_like(self.p)
        self.v = torch.zeros_like(self.p)
        self._lookup = lookup
        self.scratch = None
        self._build_segs()
        self.step_dev = torch.zeros(1, dtype=torch.int64, device=dev)
        self._built = True

    def _group_signature(self):
        return tuple((float(g["lr"]), float(g["weight_decay"]), len(g["params"])) for g in self.param_groups)

    def _build_segs(self):
        """device chunk table {offset, count, tensor, lr, weight_decay}; rebuilt whenever a param group's lr or
        weight_decay is edited (or restored by load_state_dict), as torch optimizers honour such edits"""
        import struct
        dev = self.p.device
        rows = []
        grp0 = self.param_groups[0]
        for grp in self.param_groups:
            for key in ("b1", "b2", "e", "max_grad_norm", "warmup", "t_total"):
                if grp[key] != grp0[key]:
                    raise ValueError("FusedBertAdam: %s must be the same in every param group" % key)
            for p in grp["params"]:
                off, n, _ = self._lookup[id(p)]
                rows.append((off, n, float(grp["lr"]), float(grp["weight_decay"])))
        chunk = 65536
        parts = []
        for t, (off, n, lr, wd) in enumerate(rows):
            for c0 in range(0, n, chunk):
                parts.append(struct.pack("<qiiffff", off + c0, min(chunk, n - c0), t, lr, wd, 0.0, 0.0))
        self.segs = torch.frombuffer(bytearray(b"".join(parts)), dtype=torch.uint8).to(dev)
        self.n_chunks = len(parts)
        self.n_tensors = len(rows)
        if self.scratch is None or self.scratch.numel() != self.n_tensors + 1:
            self.scratch = torch.zeros(self.n_tensors + 1, dtype=torch.float32, device=dev)
        self._sig = self._group_signature()

    # ---- checkpointing in the reference's layout (modules/optimization.py:121-128: per-parameter
    # {'step', 'next_m', 'next_v'}; main_pretrain.py:270 saves it, :389 restores it) --------------------------
    def state_dict(self):
        if not self._built:
            return super(FusedBertAdam, self).state_dict()
        step = int(self.step_dev.item())
        self.state.clear()
        if step > 0:
            for grp in self.param_groups:
                for p in grp["params"]:
                    off, n, shape = self._lookup[id(p)]
                    self.state[p] = {"step": step, "next_m": self.m[off:off + n].view(shape).clone(),
                                     "next_v": self.v[off:off + n].view(shape).clone()}
        sd = super(FusedBertAdam, self).state_dict()
        self.state.clear()
        return sd

    def load_state_dict(self, state_dict):
        super(FusedBertAdam, self).load_state_dict(state_dict)
        if not self._built:
            self._build()
        step = 0
        self.m.zero_()
        self.v.zero_()
        for p, st in list(self.state.items()):
            if id(p) not in self._lookup or "next_m" not in st:
                continue
            off, n, _ = self._lookup[id(p)]
            self.m[off:off + n].copy_(st["next_m"].reshape(-1))
            self.v[off:off + n].copy_(st["next_v"].reshape(-1))
            step = max(step, int(st["step"]))
        self.state.clear()
        self.step_dev.fill_(step)
        self._build_segs()

    def zero_grad(self, set_to_none=False):
        """Reference drivers call only `optimizer.zero_grad()` after `optimizer.step()` (main_task_retrieval.py:353,
        main_pretrain.py:345), so this must clear whatever autograd accumulates into.  Flat layout: the gradient
        buffer IS every p.grad (views; re-attached if a `model.zero_grad(set_to_none=True)` dropped them).  Compat
        layout (no `model=`): the per-parameter grads autograd/DDP own are cleared as torch.optim.Optimizer does, in
        addition to the private flat copy."""
        if not self._built:
            return super(FusedBertAdam, self).zero_grad(set_to_none=set_to_none)
        _zero(self.g)
        if self.flat is not None:
            for p, off in zip(self.flat.params, self.flat.offsets):
                if p.grad is None or p.grad.data_ptr() != self.g.data_ptr() + 4 * off:
                    p.grad = self.g[off:off + p.numel()].view(p.shape)
        else:
            super(FusedBertAdam, self).zero_grad(set_to_none=set_to_none)

    def _gather_grads(self):
        """no flat model: copy per-parameter grads into the flat gradient buffer (compat path)"""
        for p, off in zip(self._plist, self._offs):
            n = p.numel()
            if p.grad is None:
                self.g[off:off + n].zero_()
            else:
                self.g[off:off + n].copy_(p.grad.reshape(-1))

    @torch.no_grad()
    def step(self, closure=None):
        loss = closure() if closure is not None else None
        if not self._built:
            grads = {id(p): p.grad for grp in self.param_groups for p in grp["params"]}
            self._build()
            if self.flat is not None:           # first step: gradients were produced before flattening
                for p in self.flat.params:
                    gr = grads.get(id(p))
                    if gr is not None and gr.data_ptr() != p.grad.data_ptr():
                        p.grad.copy_(gr)
        if self.flat is None:
            self._gather_grads()
        if self._group_signature() != self._sig:
            self._build_segs()
        g0 = self.param_groups[0]
        payload = self.grad_payload
        if payload is not None and (payload.dtype != torch.bfloat16 or payload.numel() != self.g.numel()
                                    or payload.device != self.g.device):
            raise ValueError("FusedBertAdam.grad_payload must be a bf16 tensor shaped like the flat gradient buffer")
        call("univl_bert_adam_step" if payload is None else "univl_bert_adam_step_bf16grad", self.p.data_ptr(),
             (self.g if payload is None else payload).data_ptr(), self.m.data_ptr(), self.v.data_ptr(),
             None if self.shadow is None else self.shadow.data_ptr(), self.segs.data_ptr(), self.n_chunks,
             self.n_tensors, self.scratch.data_ptr(), self.step_dev.data_ptr(), float(g0["b1"]), float(g0["b2"]),
             float(g0["e"]), float(g0["max_grad_norm"]), self.global_clip_norm, float(g0["warmup"]),
             int(g0["t_total"]), self.grad_scale)
        if self.flat is not None:
            self.flat.arena.fresh = True
        return loss
