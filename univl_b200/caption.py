"""KV-cached caption decoding and beam search (SURVEY.md §8f#3).

The reference's caption evaluation (main_task_caption.py:434-517) calls `model.decoder_caption` once per generated
token on the FULL prefix: every step re-runs the 2-layer cross encoder on n_inst * n_beam copies of the (text, video)
pair and the 3 decoder layers on all t prefix tokens, then keeps only the last position's logits — O(L^2) decoder work
and L * n_beam redundant cross-encoder passes.  Here, per batch of instances:

  * the cross encoder runs ONCE per instance; the key/value projections of every decoder layer's encoder-attention are
    computed ONCE per instance and shared by its beams — the n_beam hypotheses of an instance are the Sq = n_beam query
    rows of one attention "sequence" over the instance's S_e encoder keys, so nothing is ever `repeat`ed;
  * each decoder layer keeps a self-attention K/V cache [n_inst * n_beam, L_max, 2H]; a step projects only the NEW
    token (q | k | v in one GEMM), appends its k | v at position t, and attends with Sq = 1 over the cache under a
    (position <= t) mask; beam reordering is an index_select of the cache rows by the beams' back-pointers;
  * the vocabulary projection runs on the n_inst * n_beam last-token rows only.

Same kernels as the training path (C ABI: univl_gemm_bf16, univl_attention_fwd, univl_layernorm_fwd,
univl_embed_text_fwd); arithmetic per token is identical to `decoder_caption` on the full prefix (tested to bf16
tolerance against it).  The beam bookkeeping restates `modules/beam.py` (Beam.advance :63-87: scores summed with the
previous beam scores except at the first step, top-k over beam x vocabulary, back-pointers, finished when the top
hypothesis ends in [SEP]) in batched tensor form.
"""
import os

import torch

from . import ops
from . import runtime as rt

BF16 = torch.bfloat16
I32 = torch.int32

DECODE_CACHE_MODES = ("off", "prefix")


def decode_cache_mode():
    """UNIVL_DECODE_CACHE, read on every `UniVL.decoder_caption` call: "off" (default) computes every call on its full
    prefix; "prefix" serves the calls through the model's PrefixDecodeCache.  An environment variable, so that the
    caption driver picks it up unchanged."""
    value = os.environ.get("UNIVL_DECODE_CACHE", "off")
    if value not in DECODE_CACHE_MODES:
        raise ValueError("UNIVL_DECODE_CACHE must be one of %s, got %r" % ("/".join(DECODE_CACHE_MODES), value))
    return value


class CachedCaptionDecoder:
    """Incremental decoder state for `n_inst` instances x `n_beam` hypotheses."""

    def __init__(self, model, sequence_output, visual_output, input_mask, video_mask, n_beam, max_len):
        self.model = model
        dec = model.decoder
        self.dec = dec
        self.n_inst = sequence_output.shape[0]
        self.n_beam = int(n_beam)
        self.max_len = int(max_len)
        self.H = sequence_output.shape[-1]
        dev = sequence_output.device
        self.device = dev
        input_mask = input_mask.reshape(self.n_inst, -1).long().contiguous()
        video_mask = video_mask.reshape(self.n_inst, -1).long().contiguous()
        with rt.use_model(model, dev):
            seq2d = sequence_output.to(BF16).reshape(-1, self.H).contiguous()
            vis2d = visual_output.to(BF16).reshape(-1, self.H).contiguous()
            # reference modeling.py:393-399: decoder attends to the cross-encoder output of (text, video)
            self.enc2d, _, self.Se = model._cross_pairs(seq2d, vis2d, input_mask, video_mask, False)
            arena = rt.current()
            self.enc_mask = ops.MaskSpec(input_mask, video_mask)
            self.enc_kv = []
            for layer in dec.decoder.layer:
                att = layer.enc_attn.att
                wqkv = arena.bf16_qkv(att.query.weight, att.key.weight, att.value.weight)
                self.enc_kv.append(ops.linear_fwd(self.enc2d, wqkv[self.H:], rt.packed_bias(att.key.bias, att.value.bias)))
        rows = self.n_inst * self.n_beam
        self.cache = [torch.zeros(rows, self.max_len, 2 * self.H, dtype=BF16, device=dev) for _ in dec.decoder.layer]
        self.t = 0
        self.active = torch.arange(self.n_inst, device=dev)      # instance index of every active cache slot

    # ------------------------------------------------------------------------------------------------------
    def select(self, keep_positions):
        """keep only these active positions (finished instances leave the batch, main_task_caption.py:400-421)"""
        idx = torch.as_tensor(keep_positions, device=self.device, dtype=torch.long)
        rows = (idx.unsqueeze(1) * self.n_beam + torch.arange(self.n_beam, device=self.device)).reshape(-1)
        self.cache = [c.index_select(0, rows) for c in self.cache]
        self.active = self.active.index_select(0, idx)

    def reorder(self, origin):
        """origin [n_active, n_beam]: beam j of an instance continues hypothesis origin[i, j] of the previous step"""
        n = origin.shape[0]
        rows = (torch.arange(n, device=self.device).unsqueeze(1) * self.n_beam + origin).reshape(-1)
        self.cache = [c.index_select(0, rows) for c in self.cache]

    def step(self, tokens):
        """tokens int64 [n_active * n_beam]: the token at position self.t of every hypothesis.
        -> fp32 logits [n_active * n_beam, vocab] for position self.t + 1"""
        dec, H, t = self.dec, self.H, self.t
        if t >= self.max_len:
            raise RuntimeError("CachedCaptionDecoder: sequence longer than max_len=%d" % self.max_len)
        n_act = self.active.shape[0]
        rows = n_act * self.n_beam
        model = self.model
        with rt.use_model(model, self.device):
            arena = rt.current()
            emb = dec.embeddings
            # word + position[t] -> LayerNorm (reference module_decoder.py:309-320); the position table view starts at row t
            x = ops.EmbedTextFn.apply(tokens.reshape(rows, 1).contiguous(), None, emb.word_embeddings.weight,
                                      emb.position_embeddings.weight[t:], None, emb.LayerNorm.weight,
                                      emb.LayerNorm.bias, 0.0, False)
            pos_mask = (torch.arange(self.max_len, device=self.device) <= t).long().unsqueeze(0).expand(rows, -1)
            slf_mask = ops.MaskSpec(pos_mask.contiguous())
            # encoder K/V and padding masks of the ACTIVE instances (one gather per step; the full set when none left)
            all_active = n_act == self.n_inst
            if all_active:
                enc_mask = self.enc_mask
            else:
                enc_mask = ops.MaskSpec(self.enc_mask.a.index_select(0, self.active),
                                        self.enc_mask.b.index_select(0, self.active))
            for li, layer in enumerate(dec.decoder.layer):
                # ---- causal self-attention of the new token over the cache (module_decoder.py:220-247, :389-396) ----
                att, out = layer.slf_attn.att, layer.slf_attn.output
                wqkv = arena.bf16_qkv(att.query.weight, att.key.weight, att.value.weight)
                qkv = ops.linear_fwd(x, wqkv, rt.packed_bias(att.query.bias, att.key.bias, att.value.bias))
                cache = self.cache[li]
                cache[:, t] = qkv[:, H:]
                kv2d = cache.view(rows * self.max_len, 2 * H)
                ctx, _ = ops.attention_fwd(qkv[:, :H], kv2d[:, :H], kv2d[:, H:], rows, 1, self.max_len, slf_mask)
                ao = ops.linear_fwd(ctx, arena.bf16(out.dense.weight), out.dense.bias)
                x, _, _ = ops.layernorm_fwd(ao, x, out.LayerNorm.weight, out.LayerNorm.bias)
                # ---- encoder attention: the n_beam hypotheses of an instance are n_beam query rows of ONE sequence ----
                att, out = layer.enc_attn.att, layer.enc_attn.output
                wqkv = arena.bf16_qkv(att.query.weight, att.key.weight, att.value.weight)
                q = ops.linear_fwd(x, wqkv[:H], att.query.bias)
                kv = self.enc_kv[li]
                if not all_active:
                    kv = kv.view(self.n_inst, self.Se, 2 * H).index_select(0, self.active).view(-1, 2 * H)
                ctx, _ = ops.attention_fwd(q, kv[:, :H], kv[:, H:], n_act, self.n_beam, self.Se, enc_mask)
                ao = ops.linear_fwd(ctx, arena.bf16(out.dense.weight), out.dense.bias)
                x, _, _ = ops.layernorm_fwd(ao, x, out.LayerNorm.weight, out.LayerNorm.bias)
                # ---- feed-forward ----
                w1, w2 = arena.bf16(layer.intermediate.dense.weight), arena.bf16(layer.output.dense.weight)
                pre = torch.empty(rows, w1.shape[0], dtype=BF16, device=self.device)
                h = ops.linear_fwd(x, w1, layer.intermediate.dense.bias, epi=ops.EPI_GELU, aux_out=pre)
                fo = ops.linear_fwd(h, w2, layer.output.dense.bias)
                x, _, _ = ops.layernorm_fwd(fo, x, layer.output.LayerNorm.weight, layer.output.LayerNorm.bias)
            logits = dec.classifier.cls.logits(x)
        self.t += 1
        return logits


# Row fingerprints of PrefixDecodeCache: the bytes of a row as int16 times integer weights in [1, 2^16), summed in fp64.
# Every partial sum is an integer below 2^53 when a row has fewer than 2^22 int16 words, so the sums are exact in any
# order: equal rows always get equal fingerprints.  They only pick the candidate parent; equality is then checked bitwise.
HASH_WEIGHT_BITS = 16
HASH_MAX_WORDS = 1 << 22
HASH_CHUNK_ELEMS = 1 << 22          # int16 words converted to fp64 at a time
PLANES_MIN = 32                     # self-attention cache positions allocated at a fill; doubled as decoding goes on


def _int16_rows(t, rows):
    """the bytes of t [rows, ...] as int16 [rows, n] (1-byte types are widened: the values are what is compared)"""
    t = t.contiguous().reshape(rows, -1)
    if t.element_size() == 1:
        return t.to(torch.int16)
    return t.view(torch.int16)


class _Call:
    """one decoder_caption call's inputs, flattened: ids int64 [R, t], masks [R, W] / [R, F], and the int16 words of the
    four encoder inputs (sequence_output, visual_output and both masks) per row"""

    def __init__(self, seq, vis, am, vm, ids, dm, H):
        self.R, self.t = ids.shape
        self.W, self.F = am.shape[1], vm.shape[1]
        self.seq, self.vis, self.am, self.vm, self.ids, self.dm = seq, vis, am, vm, ids, dm
        self.words = [_int16_rows(x, self.R) for x in (seq, vis, am, vm)]
        self.sig = (seq.dtype, vis.dtype, am.dtype, vm.dtype, self.W, self.F, H, seq.device)


class _State:
    pass


class PrefixDecodeCache:
    """Incremental evaluation of `UniVL.decoder_caption` for a caller that asks for the logits of a whole prefix once per
    generated token, as the caption driver's beam search does (main_task_caption.py:434-517).

    A decoder row's K/V and logits are a pure function of its encoder inputs and its prefix tokens, so the cache reuses
    state only when both are bitwise equal to what it was computed from.  A call of prefix length t continues the
    previous call (of length t - 1) when every row has a parent: a previous row with the same first t - 1 tokens and
    bitwise-equal encoder inputs (the lowest such index; equal rows hold equal state).  Beam reordering and the removal
    of finished instances are then just parent maps.  The continued call decodes one token per row: the row's
    self-attention reads the K/V of its ancestors through an ancestry table of key rows (one plane of cache rows per
    position, nothing is copied when beams reorder), its encoder attention reads the valid rows of its own cross-encoder
    output, computed once at the fill, and the vocabulary projection runs on the new rows only.  Earlier positions'
    logits come from a per-position history, gathered through the ancestry table.

    Eligible calls: model.eval(), no gradients, every decoder_mask entry nonzero and t within the decoder's position
    table.  Every other call computes the full path and leaves the cache alone.  An eligible call that does not continue
    the previous one fills the cache: at t = 1 it decodes position 0 and returns that; at t > 1 it returns the full
    path's result and refills by decoding the call's t positions.  A call in which any row has no valid encoder key
    takes the full path, as does a fill of such rows.  The decision costs one device-to-host read per call.  The full
    path gets decoder_mask as int64 (the caption driver passes uint8 ones, which the default path rejects).

    The state lives on the model (PrefixDecodeCache.of), never in state_dict(), and is released by model.train()."""

    def __init__(self, model):
        self.model = model
        self.state = None
        self._weights = {}

    @staticmethod
    def of(model):
        """the cache of this very module: a `parallel_apply` replica carries a copy of the original's __dict__"""
        c = model.__dict__.get("_univl_decode_cache")
        if c is None or c.model is not model:
            c = PrefixDecodeCache(model)
            model.__dict__["_univl_decode_cache"] = c
        return c

    @staticmethod
    def release(model):
        model.__dict__.pop("_univl_decode_cache", None)

    # ------------------------------------------------------------------------------------------------------
    def logits(self, sequence_output, visual_output, attention_mask, video_mask, input_caption_ids, decoder_mask,
               shaped=False):
        """`UniVL._get_decoder_score`'s logits fp32 [R, t, vocab], incrementally where the call allows it"""
        model = self.model
        # the default path takes int64 masks only; the caption driver builds its decoder mask as uint8 ones
        full_mask = decoder_mask.long() if isinstance(decoder_mask, torch.Tensor) else decoder_mask

        def full():
            return model._get_decoder_score(sequence_output, visual_output, None, attention_mask, video_mask,
                                            input_caption_ids, full_mask, shaped=shaped)[0]

        x = self._call(sequence_output, visual_output, attention_mask, video_mask, input_caption_ids, decoder_mask,
                       shaped)
        if x is None:
            return full()
        st = self.state
        cont = st is not None and st.sig == x.sig and x.t == st.t + 1 and x.R <= st.R0
        dev = x.ids.device
        with torch.no_grad():
            mask_ok = (x.dm != 0).all()
            enc_ok = torch.cat([x.am != 0, x.vm != 0], 1).any(1).all()
            if cont:
                parent, matched, hashes = self._match(x)
            else:
                matched = torch.zeros((), dtype=torch.bool, device=dev)
            flag = int((mask_ok.long() | (enc_ok.long() << 1) | (matched.long() << 2)).item())  # the one read
        if not flag & 1:
            return full()
        if flag & 4:
            with torch.no_grad(), rt.use_model(model, dev):
                st.hash_rows = hashes
                self._advance(x.ids[:, -1], parent)
                return self._gather(x.R)
        self.state = None
        if not flag & 2:
            return full()
        if x.t == 1:
            with torch.no_grad(), rt.use_model(model, dev):
                self._fill(x)
                self._advance(x.ids[:, 0], None)
                return self._gather(x.R)
        out = full()
        with torch.no_grad(), rt.use_model(model, dev):
            self._fill(x)
            for p in range(x.t):
                self._advance(x.ids[:, p], None)
        return out

    # ------------------------------------------------------------------------------------------------------
    def _call(self, seq, vis, am, vm, ids, dm, shaped):
        """_Call of an eligible call's arguments (flattened as _get_decoder_score flattens them), else None"""
        model = self.model
        if model.training or torch.is_grad_enabled():
            return None
        if not all(isinstance(a, torch.Tensor) for a in (seq, vis, am, vm, ids, dm)):
            return None
        if shaped is False:
            am, vm = am.reshape(-1, am.shape[-1]), vm.reshape(-1, vm.shape[-1])
            ids, dm = ids.reshape(-1, ids.shape[-1]), dm.reshape(-1, dm.shape[-1])
        dec = model.decoder
        H = dec.embeddings.word_embeddings.weight.shape[1]
        dev = dec.embeddings.word_embeddings.weight.device
        if ids.dim() != 2 or am.dim() != 2 or vm.dim() != 2 or dm.shape != ids.shape or ids.dtype != torch.int64:
            return None
        R, t = ids.shape
        if R == 0 or t == 0 or t > dec.embeddings.position_embeddings.weight.shape[0]:
            return None
        if am.shape[0] != R or vm.shape[0] != R or seq.numel() != R * am.shape[1] * H or \
                vis.numel() != R * vm.shape[1] * H:
            return None
        if any(a.device != dev for a in (seq, vis, am, vm, ids, dm)):
            return None
        x = _Call(seq, vis, am, vm, ids.contiguous(), dm, H)
        if any(w.shape[1] >= HASH_MAX_WORDS for w in x.words):
            return None
        return x

    def _weight(self, i, n, device):
        key = (i, n, device)
        w = self._weights.get(key)
        if w is None:
            g = torch.Generator().manual_seed(0x5EED + i)
            w = torch.randint(1, 1 << HASH_WEIGHT_BITS, (n, 2), generator=g, dtype=torch.int64).double().to(device)
            self._weights[key] = w
        return w

    def _hash(self, words):
        """fp64 [R, 2 * len(words)] exact fingerprints of int16 rows"""
        cols = []
        for i, a in enumerate(words):
            R, n = a.shape
            w = self._weight(i, n, a.device)
            step = max(1, HASH_CHUNK_ELEMS // max(1, n))
            cols.append(torch.cat([a[r:r + step].double() @ w for r in range(0, R, step)]))
        return torch.cat(cols, 1)

    def _match(self, x):
        """-> (parent int64 [R], every row has a parent (device bool), fingerprints of the call's rows)"""
        st = self.state
        h = self._hash(x.words)
        cand = (x.ids[:, None, :-1] == st.tokens[None]).all(2) & (h[:, None] == st.hash_rows[None]).all(2)
        parent = cand.int().argmax(1)               # the lowest candidate (0 when none: `ok` is then False)
        ok = cand.any(1)
        fill_row = st.fill_of.long().index_select(0, parent)
        for new, kept in zip(x.words, st.words):
            ok = ok & (new == kept.index_select(0, fill_row)).all(1)
        return parent, ok.all(), h

    def _fill(self, x):
        """encoder side of the call's rows: cross encoder once, every decoder layer's encoder K/V once, the valid key
        lists; an empty self-attention cache"""
        model = self.model
        dec = model.decoder
        H = x.sig[6]
        arena = rt.current()
        dev = x.ids.device
        seq2d = x.seq.to(BF16).reshape(-1, H).contiguous()
        vis2d = x.vis.to(BF16).reshape(-1, H).contiguous()
        am, vm = x.am.contiguous(), x.vm.contiguous()
        enc2d, _, Se = model._cross_pairs(seq2d, vis2d, am, vm, False)
        st = _State()
        st.sig, st.R0, st.t = x.sig, x.R, 0
        st.enc_kv = []
        for layer in dec.decoder.layer:
            att = layer.enc_attn.att
            wqkv = arena.bf16_qkv(att.query.weight, att.key.weight, att.value.weight)
            st.enc_kv.append(ops.linear_fwd(enc2d, wqkv[H:], rt.packed_bias(att.key.bias, att.value.bias)))
        del enc2d
        # key list of row f: its valid encoder rows f * Se + s, ascending (cumsum + scatter, no nonzero())
        valid = torch.cat([am != 0, vm != 0], 1)
        slot = torch.where(valid, torch.cumsum(valid, 1) - 1, Se)
        table = torch.zeros(x.R, Se + 1, dtype=I32, device=dev)
        table.scatter_(1, slot, torch.arange(x.R * Se, dtype=I32, device=dev).view(x.R, Se))
        st.enc_rows, st.enc_n = table[:, :Se], valid.sum(1).to(I32)
        st.words = [w.clone() for w in x.words]
        st.hash_rows = self._hash(st.words)
        st.fill_of = torch.arange(x.R, dtype=I32, device=dev)
        st.anc = torch.empty(x.R, 0, dtype=I32, device=dev)         # key row of every ancestor: p * R0 + its slot
        st.slots = torch.empty(x.R, 0, dtype=torch.int64, device=dev)  # row of every ancestor in its step's history
        st.tokens = torch.empty(x.R, 0, dtype=torch.int64, device=dev)
        st.hist = []
        cap = min(PLANES_MIN, dec.embeddings.position_embeddings.weight.shape[0])
        st.planes = [torch.empty(cap, x.R, 2 * H, dtype=BF16, device=dev) for _ in dec.decoder.layer]
        self.state = st

    def _advance(self, tokens, parent):
        """decode the token at position st.t of every row; parent int64 [R] (previous row of each row) or None (the
        rows continue themselves)"""
        st = self.state
        dec = self.model.decoder
        arena = rt.current()
        H = st.sig[6]
        R, p, dev = tokens.shape[0], st.t, tokens.device
        if parent is not None:
            st.anc, st.slots = st.anc.index_select(0, parent), st.slots.index_select(0, parent)
            st.fill_of, st.tokens = st.fill_of.index_select(0, parent), st.tokens.index_select(0, parent)
        here = torch.arange(R, device=dev)
        st.anc = torch.cat([st.anc, (here + p * st.R0).to(I32)[:, None]], 1)
        st.slots = torch.cat([st.slots, here[:, None]], 1)
        st.tokens = torch.cat([st.tokens, tokens[:, None]], 1)
        cap = st.planes[0].shape[0]
        if p >= cap:
            for li, old in enumerate(st.planes):
                new = torch.empty(min(2 * cap, dec.embeddings.position_embeddings.weight.shape[0]), *old.shape[1:],
                                  dtype=BF16, device=dev)
                new[:cap] = old
                st.planes[li] = new
        emb = dec.embeddings
        x = ops.EmbedTextFn.apply(tokens.reshape(R, 1).contiguous(), None, emb.word_embeddings.weight,
                                  emb.position_embeddings.weight[p:], None, emb.LayerNorm.weight, emb.LayerNorm.bias,
                                  0.0, False)
        n_self = torch.full((R,), p + 1, dtype=I32, device=dev)
        for li, layer in enumerate(dec.decoder.layer):
            # ---- self-attention of the new token over its ancestors' cache rows ----
            att, out = layer.slf_attn.att, layer.slf_attn.output
            wqkv = arena.bf16_qkv(att.query.weight, att.key.weight, att.value.weight)
            qkv = ops.linear_fwd(x, wqkv, rt.packed_bias(att.query.bias, att.key.bias, att.value.bias))
            plane = st.planes[li]
            plane[p, :R] = qkv[:, H:]
            ctx = ops.attention_decode_fwd(qkv[:, :H], plane.view(-1, 2 * H), st.anc, n_self)
            ao = ops.linear_fwd(ctx, arena.bf16(out.dense.weight), out.dense.bias)
            x, _, _ = ops.layernorm_fwd(ao, x, out.LayerNorm.weight, out.LayerNorm.bias)
            # ---- encoder attention over the valid rows of the row's own cross-encoder output ----
            att, out = layer.enc_attn.att, layer.enc_attn.output
            wqkv = arena.bf16_qkv(att.query.weight, att.key.weight, att.value.weight)
            q = ops.linear_fwd(x, wqkv[:H], att.query.bias)
            ctx = ops.attention_decode_fwd(q, st.enc_kv[li], st.enc_rows, st.enc_n, st.fill_of)
            ao = ops.linear_fwd(ctx, arena.bf16(out.dense.weight), out.dense.bias)
            x, _, _ = ops.layernorm_fwd(ao, x, out.LayerNorm.weight, out.LayerNorm.bias)
            # ---- feed-forward ----
            w1, w2 = arena.bf16(layer.intermediate.dense.weight), arena.bf16(layer.output.dense.weight)
            pre = torch.empty(R, w1.shape[0], dtype=BF16, device=dev)
            h = ops.linear_fwd(x, w1, layer.intermediate.dense.bias, epi=ops.EPI_GELU, aux_out=pre)
            fo = ops.linear_fwd(h, w2, layer.output.dense.bias)
            x, _, _ = ops.layernorm_fwd(fo, x, layer.output.LayerNorm.weight, layer.output.LayerNorm.bias)
        st.hist.append(dec.classifier.cls.logits(x))
        st.t += 1

    def _gather(self, R):
        """fp32 [R, t, vocab]: position p of row r is the logits its ancestor at position p was decoded with"""
        st = self.state
        V = st.hist[0].shape[1]
        out = torch.empty((R, st.t, V), dtype=torch.float32, device=st.hist[0].device)
        for p, h in enumerate(st.hist):
            out[:, p] = h.index_select(0, st.slots[:, p])
        return out


@torch.no_grad()
def beam_search(model, sequence_output, visual_output, input_mask, video_mask, max_words, n_beam=5, bos=101, eos=102):
    """Caption beam search with the semantics of the reference loop (main_task_caption.py:434-517 with modules/beam.py)
    on the KV-cached decoder.  sequence_output [n, W, H], visual_output [n, F, H] (from get_sequence_visual_output).
    -> (hypotheses: list over instances of the best token-id list (without [CLS]), scores: list of floats)"""
    if model.training:
        raise RuntimeError("beam_search: call model.eval() first")
    dev = sequence_output.device
    n_inst = sequence_output.shape[0]
    dec = CachedCaptionDecoder(model, sequence_output, visual_output, input_mask, video_mask, n_beam, max_words)
    scores = torch.zeros(n_inst, n_beam, device=dev)                  # Beam.scores
    next_ys = [torch.full((n_inst, n_beam), bos, dtype=torch.long, device=dev)]
    prev_ks = []
    done = torch.zeros(n_inst, dtype=torch.bool, device=dev)
    active = torch.arange(n_inst, device=dev)                         # instance ids still decoding, in cache order
    for step in range(1, max_words + 1):
        tokens = next_ys[-1].index_select(0, active).reshape(-1)
        logits = dec.step(tokens)
        word_prob = torch.log_softmax(logits, dim=1).view(active.shape[0], n_beam, -1)
        V = word_prob.shape[-1]
        if step == 1:
            beam_lk = word_prob[:, 0]                                 # Beam.advance: only hypothesis 0 exists at first
        else:
            beam_lk = (word_prob + scores.index_select(0, active).unsqueeze(-1)).reshape(active.shape[0], -1)
        best, best_id = beam_lk.topk(n_beam, dim=1, largest=True, sorted=True)
        prev_k = best_id // V
        word = best_id - prev_k * V
        full_k = torch.zeros(n_inst, n_beam, dtype=torch.long, device=dev)
        full_w = torch.zeros(n_inst, n_beam, dtype=torch.long, device=dev)
        full_k[active], full_w[active] = prev_k, word
        scores[active] = best
        prev_ks.append(full_k)
        next_ys.append(full_w)
        finished = word[:, 0] == eos                                  # top-of-beam is [SEP]
        done[active[finished]] = True
        keep = (~finished).nonzero().flatten()
        if keep.numel() == 0:
            break
        dec.reorder(prev_k)
        if keep.numel() != active.numel():
            dec.select(keep)
            active = active.index_select(0, keep)
    # best hypothesis per instance: walk the back-pointers from the top-scoring beam (Beam.sort_scores / get_hypothesis)
    order = scores.argsort(dim=1, descending=True)
    hyps, outs = [], []
    ks = torch.stack(prev_ks).cpu()        # [steps, n_inst, n_beam]
    ys = torch.stack(next_ys).cpu()        # [steps + 1, n_inst, n_beam]
    order_c, scores_c = order.cpu(), scores.cpu()
    n_steps = ks.shape[0]
    # an instance stops advancing at the step it finished: later rows of ks / ys for it are zeros and are not walked
    last = torch.full((n_inst,), n_steps, dtype=torch.long)
    for i in range(n_inst):
        for s in range(n_steps):
            if int(ys[s + 1, i, 0]) == eos:
                last[i] = s + 1
                break
    for i in range(n_inst):
        k = int(order_c[i, 0])
        hyp = []
        for j in range(int(last[i]) - 1, -1, -1):
            hyp.append(int(ys[j + 1, i, k]))
            k = int(ks[j, i, k])
        hyps.append(hyp[::-1])
        outs.append(float(scores_c[i, int(order_c[i, 0])]))
    return hyps, outs
