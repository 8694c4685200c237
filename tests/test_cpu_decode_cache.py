"""CPU: the UNIVL_DECODE_CACHE switch, PrefixDecodeCache's parent matching and call rules (univl_b200/caption.py), and
the host-side Beam (univl_b200/modules/beam.py) against the reference's Beam."""
import contextlib
import importlib.util
import os
import types

import pytest
import torch

from univl_b200 import caption
from univl_b200.caption import PrefixDecodeCache, _Call, _State, decode_cache_mode

H = 768


def test_switch_values(monkeypatch):
    monkeypatch.delenv("UNIVL_DECODE_CACHE", raising=False)
    assert decode_cache_mode() == "off"
    for v in ("off", "prefix"):
        monkeypatch.setenv("UNIVL_DECODE_CACHE", v)
        assert decode_cache_mode() == v
    for v in ("on", "", "Prefix", "1"):
        monkeypatch.setenv("UNIVL_DECODE_CACHE", v)
        with pytest.raises(ValueError, match="UNIVL_DECODE_CACHE"):
            decode_cache_mode()


def _fake_model(positions=16):
    emb = types.SimpleNamespace(word_embeddings=types.SimpleNamespace(weight=torch.zeros(50, H)),
                                position_embeddings=types.SimpleNamespace(weight=torch.zeros(positions, H)))
    model = types.SimpleNamespace(training=False, decoder=types.SimpleNamespace(embeddings=emb), full_calls=0)

    def full(seq, vis, ids, am, vm, cap, dm, shaped=False):
        model.full_calls += 1
        return torch.full((cap.shape[0], cap.shape[1], 3), -1.0), ()
    model._get_decoder_score = full
    return model


def _encoder(n, W=4, F=3, seed=0):
    g = torch.Generator().manual_seed(seed)
    seq = torch.randn(n, W, H, generator=g).to(torch.bfloat16)
    vis = torch.randn(n, F, H, generator=g).to(torch.bfloat16)
    am = (torch.rand(n, W, generator=g) < 0.8).long()
    am[:, 0] = 1
    vm = (torch.rand(n, F, generator=g) < 0.8).long()
    return seq, vis, am, vm


def _state(cache, x):
    """the state a fill of call x leaves, bookkeeping only"""
    st = _State()
    st.sig, st.R0, st.t = x.sig, x.R, 0
    st.words = [w.clone() for w in x.words]
    st.hash_rows = cache._hash(st.words)
    st.fill_of = torch.arange(x.R, dtype=torch.int32)
    st.tokens = torch.empty(x.R, 0, dtype=torch.long)
    return st


def _loop_parents(new_words, new_ids, kept_words, fill_of, prev_tokens):
    """parent of every row by a Python loop, or None when a row has none"""
    out = []
    for r in range(new_ids.shape[0]):
        found = None
        for q in range(prev_tokens.shape[0]):
            f = int(fill_of[q])
            if torch.equal(new_ids[r, :-1], prev_tokens[q]) and \
                    all(torch.equal(a[r], b[f]) for a, b in zip(new_words, kept_words)):
                found = q
                break
        out.append(found)
    return out


def _check_match(cache, x):
    parent, ok, h = cache._match(x)
    st = cache.state
    want = _loop_parents(x.words, x.ids, st.words, st.fill_of, st.tokens)
    assert bool(ok) == all(p is not None for p in want)
    for r, p in enumerate(want):
        if p is not None:
            assert int(parent[r]) == p, (r, int(parent[r]), p)
    return want


def test_parent_matching_against_a_python_loop():
    cache = PrefixDecodeCache(_fake_model())
    n_inst, n_bm, t = 4, 3, 3
    seq, vis, am, vm = _encoder(n_inst)
    seq[3], vis[3], am[3], vm[3] = seq[1], vis[1], am[1], vm[1]       # instances 1 and 3 have equal inputs
    rep = lambda a: a.repeat_interleave(n_bm, 0)
    R = n_inst * n_bm
    g = torch.Generator().manual_seed(1)
    prev = torch.randint(1000, 2000, (R, t), generator=g)
    prev[:, 0] = 101
    prev[9:12] = prev[3:6]                                            # and the same prefixes: duplicate candidates
    x0 = _Call(rep(seq), rep(vis), rep(am), rep(vm), prev, torch.ones_like(prev), H)
    cache.state = _state(cache, x0)
    cache.state.tokens = prev.clone()
    cache.state.fill_of = torch.randperm(R, generator=g).to(torch.int32)   # rows moved since the fill
    fo = cache.state.fill_of.long()
    cache.state.hash_rows = cache.state.hash_rows[fo]                  # fingerprints of the previous rows
    kept = lambda a: rep(a)[fo]                                        # the encoder inputs of the previous rows

    def call(rows, words=None):
        rows = torch.as_tensor(rows)
        ids = torch.cat([prev[rows], torch.randint(1000, 2000, (len(rows), 1), generator=g)], 1)
        e = [kept(a)[rows] for a in (seq, vis, am, vm)]
        return _Call(*e, ids, torch.ones_like(ids), H)

    # reordered rows
    perm = torch.randperm(R, generator=g)
    want = _check_match(cache, call(perm))
    assert all(p is not None for p in want)
    # instance 2 removed
    want = _check_match(cache, call([r for r in range(R) if r // n_bm != 2]))
    assert all(p is not None for p in want)
    # duplicates: with the rows in fill order, rows of instance 3 match rows of instance 1 first (lowest index)
    fresh = _state(cache, x0)
    fresh.tokens = prev.clone()
    cache.state, moved = fresh, cache.state
    x = _Call(*[rep(a)[9:12] for a in (seq, vis, am, vm)], torch.cat([prev[9:12], prev[9:12, :1]], 1),
              torch.ones(3, t + 1, dtype=torch.long), H)
    assert _check_match(cache, x) == [3, 4, 5]
    cache.state = moved
    # no match: a foreign token, and a flipped bit in one encoder row
    x = call(perm)
    x.ids[4, 1] += 1
    want = _check_match(cache, x)
    assert want[4] is None and sum(p is None for p in want) == 1
    x = call(perm)
    x.seq = x.seq.clone()
    x.seq.view(torch.int16)[7, 2, 5] ^= 1
    x.words[0] = x.seq.reshape(R, -1).view(torch.int16)
    want = _check_match(cache, x)
    assert want[7] is None and sum(p is None for p in want) == 1


class _Recorder:
    """PrefixDecodeCache with the device work replaced by the bookkeeping it does"""

    def __init__(self, monkeypatch, positions=16):
        self.model = _fake_model(positions)
        self.cache = PrefixDecodeCache.of(self.model)
        self.log = []
        monkeypatch.setattr(caption.rt, "use_model", lambda m, d: contextlib.nullcontext())
        monkeypatch.setattr(self.cache, "_fill", self._fill)
        monkeypatch.setattr(self.cache, "_advance", self._advance)
        monkeypatch.setattr(self.cache, "_gather", lambda R: torch.full((R, self.cache.state.t, 3), 1.0))

    def _fill(self, x):
        self.log.append("fill")
        self.cache.state = _state(self.cache, x)

    def _advance(self, tokens, parent):
        self.log.append("advance")
        st = self.cache.state
        if parent is not None:
            st.tokens, st.fill_of = st.tokens[parent], st.fill_of[parent]
        st.tokens = torch.cat([st.tokens, tokens[:, None]], 1)
        st.t += 1

    def __call__(self, enc, ids, mask=None):
        self.log = []
        self.model.full_calls = 0
        out = self.cache.logits(*enc, ids, torch.ones_like(ids) if mask is None else mask, shaped=True)
        path = "full" if float(out.view(-1)[0]) < 0 else "cache"
        return path, self.log, self.model.full_calls


def test_call_rules(monkeypatch):
    rec = _Recorder(monkeypatch)
    seq, vis, am, vm = _encoder(6)
    enc = (seq, vis, am, vm)
    ids = torch.randint(1000, 2000, (6, 8))
    ids[:, 0] = 101
    with torch.no_grad():
        assert rec(enc, ids[:, :1]) == ("cache", ["fill", "advance"], 0)              # t = 1 fills
        assert rec(enc, ids[:, :2]) == ("cache", ["advance"], 0)                      # t + 1 continues
        assert rec(enc, ids[:, :2]) == ("full", ["fill", "advance", "advance"], 1)    # not t + 1: full path, refill
        assert rec(enc, ids[:, :3]) == ("cache", ["advance"], 0)
        mask = torch.ones(6, 4, dtype=torch.long)
        mask[2, 3] = 0
        assert rec(enc, ids[:, :4], mask) == ("full", [], 1)                           # a zero in decoder_mask
        assert rec(enc, ids[:, :4]) == ("cache", ["advance"], 0)                       # ... left the cache alone
        foreign = ids[:, :5].clone()
        foreign[1, 2] += 1
        assert rec(enc, foreign) == ("full", ["fill"] + ["advance"] * 5, 1)           # no parent: refill
        rec.model.training = True
        assert rec(enc, ids[:, :1]) == ("full", [], 1)                                 # training mode
        rec.model.training = False
        assert rec(enc, ids[:, :1]) == ("cache", ["fill", "advance"], 0)
        long_ids = torch.full((6, 17), 101, dtype=torch.long)
        assert rec(enc, long_ids) == ("full", [], 1)                                   # past the position table
        am0 = am.clone()
        vm0 = vm.clone()
        am0[4], vm0[4] = 0, 0
        assert rec((seq, vis, am0, vm0), ids[:, :1]) == ("full", [], 1)                # a row without encoder keys
        assert rec.cache.state is None
        assert rec(enc, ids[:, :1].repeat(2, 1)[:6]) == ("cache", ["fill", "advance"], 0)
        assert rec((seq[:5], vis[:5], am[:5], vm[:5]), torch.cat([ids[:5, :1], ids[:5, 1:2]], 1)) == \
            ("cache", ["advance"], 0)                                                  # fewer rows continue
        assert rec(enc, ids[:, :3]) == ("full", ["fill"] + ["advance"] * 3, 1)         # a row that left: no parent
    assert rec(enc, ids[:, :4]) == ("full", [], 1)                                     # gradients enabled


def test_cache_belongs_to_its_module():
    model = _fake_model()
    c = PrefixDecodeCache.of(model)
    assert PrefixDecodeCache.of(model) is c
    replica = types.SimpleNamespace(**model.__dict__)          # what nn.parallel.replicate's __dict__ copy gives
    assert PrefixDecodeCache.of(replica) is not c
    PrefixDecodeCache.release(model)
    assert "_univl_decode_cache" not in model.__dict__


# ---------------------------------------------------------------------------------------------------------------------
# host Beam against the reference's
# ---------------------------------------------------------------------------------------------------------------------
def _reference_beam():
    from oracle import build_ref
    root = build_ref.ref_root()
    if root is None or not os.path.exists(os.path.join(root, "modules", "beam.py")):
        pytest.skip("reference checkout not staged (oracle/build_ref.py)")
    spec = importlib.util.spec_from_file_location("_reference_beam", os.path.join(root, "modules", "beam.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.Beam


class _Tokenizer:
    vocab = {"[PAD]": 0, "[UNK]": 100, "[CLS]": 101, "[SEP]": 102}


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
@pytest.mark.parametrize("tokenizer", [None, _Tokenizer()], ids=["constants", "tokenizer"])
def test_host_beam_matches_the_reference_beam(seed, tokenizer):
    from univl_b200.modules.beam import Beam
    RefBeam = _reference_beam()
    size, V, steps = 5, 120, 14
    g = torch.Generator().manual_seed(seed)
    eos = 102 if tokenizer is not None else 3
    ref, got = RefBeam(size, device="cpu", tokenizer=tokenizer), Beam(size, device="cpu", tokenizer=tokenizer)
    for step in range(steps):
        logits = torch.randn(size, V, generator=g) * 3
        if step == 6 + seed:
            logits[:, eos] += 20          # [SEP] on top: the beam finishes
        word_prob = torch.log_softmax(logits, 1)
        done_ref, done_got = ref.advance(word_prob.clone()), got.advance(word_prob.clone())
        assert done_ref == done_got == ref.done == got.done
        assert torch.equal(ref.scores, got.scores)
        assert all(torch.equal(a, b) for a, b in zip(ref.next_ys, got.next_ys)) and len(ref.next_ys) == len(got.next_ys)
        assert all(torch.equal(a, b) for a, b in zip(ref.prev_ks, got.prev_ks))
        assert all(torch.equal(a, b) for a, b in zip(ref.all_scores, got.all_scores))
        assert torch.equal(ref.get_current_state(), got.get_current_state())
        assert torch.equal(ref.get_current_origin(), got.get_current_origin())
        for k in range(size):
            assert ref.get_hypothesis(k) == got.get_hypothesis(k)
        s_ref, i_ref = ref.sort_scores()
        s_got, i_got = got.sort_scores()
        assert torch.equal(s_ref, s_got) and torch.equal(i_ref, i_got)
        assert [ref.get_hypothesis(i) for i in i_ref[:1]] == [got.get_hypothesis(i) for i in i_got[:1]]
        if done_ref:
            break
    assert ref.done, "the test sequence must reach [SEP]"
    fresh_ref, fresh_got = RefBeam(size, device="cpu", tokenizer=tokenizer), Beam(size, device="cpu", tokenizer=tokenizer)
    assert torch.equal(fresh_ref.get_current_state(), fresh_got.get_current_state())
