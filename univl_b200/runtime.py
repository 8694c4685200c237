"""Per-model device runtime: bf16 weight arena, dropout RNG streams, kernel-launch counter.

The fp32 `nn.Parameter`s keep the reference's names, shapes and tying (SURVEY.md Appendix A); the tensor-core
kernels consume bf16 copies that live in ONE flat arena per model.  The copies are derived state — never in
`state_dict()` — refreshed by a single multi-tensor cast launch at each top-level entry (the reference's BertAdam
updates weights through `p.data`, which bumps no version counter, so staleness cannot be detected cheaply), unless a
fused optimizer step that writes the arena itself has marked it fresh.  query/key/value weights of one attention
block are laid out adjacently so the fused QKV projection reads them as one [2304, 768] matrix without a repack.
"""
import threading

import torch

from . import lib

_tls = threading.local()
_launches = [0]


def count_launches(n=1):
    _launches[0] += n


def launch_count():
    return _launches[0]


def stream_ptr():
    return torch.cuda.current_stream().cuda_stream


def call(name, *args):
    """C-ABI call on the current stream (the stream argument is always last)."""
    count_launches()
    return lib.call(name, *args, stream_ptr())


def ptr(t):
    return None if t is None else t.data_ptr()


def reserve_sms(n):
    """SMs a concurrent collective occupies while the kernels enqueued from now on run (include/univl_b200.h
    univl_set_reserved_sms): persistent grids shrink to the free SMs.  Captured graphs keep the grids they were built with."""
    lib.call("univl_set_reserved_sms", int(n))


class WeightArena:
    """bf16 shadow copies of every >=2-D parameter of a module tree, in one flat buffer."""

    def __init__(self, root):
        self.root = root
        self.device = None
        self.entries = []      # (param, offset, numel)
        self.by_id = {}        # id(param) -> (offset, shape)
        self.packed = {}       # (id(q), id(k), id(v)) -> (offset, rows, cols)
        self.buf = None
        self.table = None
        self._ptrs = None
        self.fresh = False
        # dropout RNG: device-resident {seed, epoch}; kernels draw Philox(seed, stream_id + (epoch << 20), element).
        # The epoch is advanced on the device at every training-mode entry, so a captured CUDA graph replays with
        # fresh masks while stream ids (position of the dropout site inside a step) stay launch constants.
        self.rng_state = None
        self.stream_counter = 0
        self.epoch_host = 0   # host mirror of the number of begin_step() calls (detects stale-mask backward passes)

    @property
    def seed(self):
        """device pointer of the RNG state (the value the kernels' `rng_state` argument takes)"""
        if self.rng_state is None:
            s = int(torch.initial_seed()) & 0x7FFFFFFFFFFFFFFF
            self.rng_state = torch.tensor([s, 0], dtype=torch.int64, device=self.device)
        return self.rng_state.data_ptr()

    def begin_step(self):
        self.stream_counter = 0
        self.epoch_host += 1
        if self.device is not None:
            call("univl_rng_advance", self.seed)

    def check_epoch(self, epoch, p):
        """Backward kernels regenerate dropout masks from the device epoch CURRENT when they run.  A second training
        forward before the first one's backward (loss1 = model(a); loss2 = model(b); (loss1 + loss2).backward(), or
        a retained graph) would silently regenerate different masks for the first forward: refuse instead."""
        if p > 0.0 and epoch != self.epoch_host:
            raise RuntimeError(
                "univl_b200: backward of a training forward from dropout epoch %d runs at epoch %d — dropout masks "
                "are regenerated from the device RNG epoch, so each training forward must be followed by its backward "
                "before the next training forward (or use model.eval() / p = 0 for the extra passes)"
                % (epoch, self.epoch_host))

    # ---- layout -----------------------------------------------------------------------------------------
    def _build(self, device):
        seen = set()
        order = []
        # attention blocks first: q, k, v weights adjacent
        for mod in self.root.modules():
            trio = getattr(mod, "_qkv_modules", None)
            if trio is None:
                continue
            ws = [m.weight for m in trio()]
            if all(id(w) not in seen for w in ws):
                for w in ws:
                    seen.add(id(w))
                    order.append(w)
                self.packed[tuple(id(w) for w in ws)] = len(order) - 3
        for p in self.root.parameters():
            if id(p) in seen or p.dim() < 2:
                continue
            seen.add(id(p))
            order.append(p)
        off = 0
        offsets = []
        for p in order:
            offsets.append(off)
            off += (p.numel() + 63) // 64 * 64  # 128-byte aligned slots
        self.buf = torch.empty(off, dtype=torch.bfloat16, device=device)
        self.entries = [(p, o, p.numel()) for p, o in zip(order, offsets)]
        self.by_id = {id(p): (o, tuple(p.shape)) for p, o in zip(order, offsets)}
        for key, first in list(self.packed.items()):
            p0 = order[first]
            contiguous = all(offsets[first + i + 1] == offsets[first + i] + order[first + i].numel() for i in range(2))
            assert contiguous, "qkv weights must be adjacent in the arena"
            self.packed[key] = (offsets[first], 3 * p0.shape[0], p0.shape[1])
        self.device = device
        self._ptrs = None

    def _sync_table(self):
        ptrs = [p.data_ptr() for p, _, _ in self.entries]
        if ptrs == self._ptrs:
            return
        base = self.buf.data_ptr()
        rows = [[pp, base + 2 * o, n] for pp, (_, o, n) in zip(ptrs, self.entries)]
        # uint64 values fit int64 for device addresses
        self.table = torch.tensor(rows, dtype=torch.int64).to(self.device)
        self._ptrs = ptrs

    def prepare(self, device):
        if self.buf is None or self.device != device:
            self._build(device)
        for p, _, _ in self.entries:
            if p.device != device:
                raise RuntimeError("univl_b200: parameters moved off %s; call model.to(device) before use" % device)
            if p.dtype != torch.float32:
                raise RuntimeError("univl_b200: parameters must stay fp32 (got %s)" % p.dtype)
        if not self.fresh and self.entries:
            self._sync_table()
            call("univl_multi_cast_f32_to_bf16", self.table.data_ptr(), len(self.entries), 16)
        self.fresh = False

    # ---- lookup ------------------------------------------------------------------------------------------
    def bf16(self, param):
        off, shape = self.by_id[id(param)]
        n = 1
        for s in shape:
            n *= s
        return self.buf[off:off + n].view(shape)

    def bf16_qkv(self, q, k, v):
        off, rows, cols = self.packed[(id(q), id(k), id(v))]
        return self.buf[off:off + rows * cols].view(rows, cols)

    def next_stream(self):
        self.stream_counter += 1
        return self.stream_counter


def arena_of(root):
    """The arena cached on `root`.  `nn.parallel.replicate` (the reference's util.parallel_apply, util.py:22) builds
    replicas with `replica.__dict__ = module.__dict__.copy()`, so a replica can carry the ORIGINAL model's arena (its
    by_id / root refer to the cuda:0 parameters): the cache is valid only when it was built for this very module."""
    a = root.__dict__.get("_univl_arena")
    if a is None or a.root is not root:
        a = WeightArena(root)
        root.__dict__["_univl_arena"] = a
    return a


class use_model:
    """Context manager for a top-level entry: prepares the arena of `root` on `device` and makes it current."""

    def __init__(self, root, device):
        self.root, self.device = root, device

    def __enter__(self):
        if self.device.type != "cuda":
            raise RuntimeError(
                "univl_b200 runs on CUDA (sm_90a) only — there is no CPU path; move the model and inputs to a "
                "H100 (got device %s)" % self.device)
        prev = getattr(_tls, "arena", None)
        self.prev = prev
        if prev is not None and prev.root is not self.root and _covers(prev, self.root):
            self.arena = prev  # nested entry of a sub-model whose parameters the outer arena already covers
        else:
            self.arena = arena_of(self.root)
            if prev is None or prev is not self.arena:
                with torch.cuda.device(self.device):
                    self.arena.prepare(self.device)
                    if prev is None and getattr(self.root, "training", False):
                        self.arena.begin_step()
        _tls.arena = self.arena
        return self.arena

    def __exit__(self, *exc):
        _tls.arena = self.prev
        return False


def _covers(arena, root):
    for p in root.parameters():
        if p.dim() >= 2 and id(p) not in arena.by_id:
            return False
    return arena.buf is not None


def set_grad_sink(flat, model):
    """register (or clear) the flat gradient buffers the backward kernels accumulate into directly"""
    model.__dict__["_univl_sink"] = flat


def current_sink():
    a = getattr(_tls, "arena", None)
    if a is None:
        return None
    sink = a.root.__dict__.get("_univl_sink")
    if sink is not None and sink.model is not a.root:   # a replica inherited the original's registration
        return None
    return sink


_side_streams = {}


def side_stream(device):
    """second stream of `device` for the branch of the model that is independent of the main one (visual encoder);
    None when disabled (UNIVL_TWO_STREAM=0).  Every fork waits for the current stream first and every join makes the
    current stream wait for it, so tensors produced on either side are ordered for the caching allocator as well."""
    import os
    if os.environ.get("UNIVL_TWO_STREAM", "1") == "0" or device.type != "cuda":
        return None
    key = (device.index if device.index is not None else torch.cuda.current_device(), threading.get_ident())
    s = _side_streams.get(key)
    if s is None:
        s = torch.cuda.Stream(device=device)
        _side_streams[key] = s
    return s


def packed_bias(*bs):
    """q/k/v projection biases as ONE [3H] vector for the fused QKV projection: a zero-copy view when the three
    parameters are adjacent in memory (the flat layout of univl_b200.optim.FlatParams), else a concatenated copy."""
    b0 = bs[0]
    n = b0.numel()
    if all(b.numel() == n and b.data_ptr() == b0.data_ptr() + 4 * n * i for i, b in enumerate(bs)):
        if b0.untyped_storage().nbytes() >= 4 * (b0.storage_offset() + n * len(bs)):
            return b0.detach().as_strided((n * len(bs),), (1,))
    return torch.cat(bs)


def current():
    a = getattr(_tls, "arena", None)
    if a is None:
        raise RuntimeError("univl_b200: no active model context (internal error)")
    return a
