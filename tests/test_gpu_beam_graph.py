"""GPU: caption beam search on the device (univl_b200.caption.GraphBeamSearch) against the eager `beam_search`.

The graph path reads the self-attention cache through univl_attention_decode_fwd and takes lse and keys from
univl_vocab_beam_topk, where `beam_search` runs a masked attention over the whole cache and torch's log_softmax / topk,
so the two agree up to rounding, not bit for bit: a step's log-probabilities differ by the bf16 roundings of the
self-attention context carried through the decoder.  E_STEP bounds that difference per step (the largest seen on an
H100 SXM was 2.7e-3; E_STEP leaves about 4x room), so a score after s steps may differ by s E_STEP.  The searches can only be compared where no candidate
choice is that close: the tests pick the classifier bias (a seeded random offset) for which every step of the eager
search separates its best from its second candidate, and its n_beam-th from its (n_beam + 1)-th, by more than
2 s E_STEP, and assert that such a bias was found, so the comparison cannot pass vacuously."""
import pytest
import torch

from tests.test_gpu_caption import _setup
from univl_b200.caption import CachedCaptionDecoder, GraphBeamSearch, beam_search

pytestmark = pytest.mark.gpu

E_STEP = 1e-2
BIAS_SIGMA = 4.0
EOS = 102


def _eager_margin(model, seq, vis, am, vm, max_words, n_beam):
    """beam_search's loop (univl_b200/caption.py) restated to record, at every step s and active instance, the gaps
    between its first and second and its n_beam-th and next candidates, divided by s; -> the smallest"""
    dec = CachedCaptionDecoder(model, seq, vis, am, vm, n_beam, max_words)
    n = seq.shape[0]
    scores = torch.zeros(n, n_beam, device="cuda")
    tokens = torch.full((n * n_beam,), 101, dtype=torch.long, device="cuda")
    active = torch.arange(n, device="cuda")
    worst = float("inf")
    for step in range(1, max_words + 1):
        wp = torch.log_softmax(dec.step(tokens), dim=1).view(active.shape[0], n_beam, -1)
        V = wp.shape[-1]
        lk = wp[:, 0] if step == 1 else (wp + scores.index_select(0, active).unsqueeze(-1)).reshape(active.shape[0], -1)
        top = lk.topk(n_beam + 1, dim=1).values
        gap = torch.minimum(top[:, 0] - top[:, 1], top[:, n_beam - 1] - top[:, n_beam])
        worst = min(worst, float(gap.min()) / step)
        best, best_id = top[:, :n_beam], lk.topk(n_beam, dim=1).indices
        prev_k, word = best_id // V, best_id % V
        scores[active] = best
        keep = (word[:, 0] != EOS).nonzero().flatten()
        if keep.numel() == 0:
            break
        dec.reorder(prev_k)
        if keep.numel() != active.numel():
            dec.select(keep)
            active, word = active.index_select(0, keep), word.index_select(0, keep)
        tokens = word.reshape(-1)
    return worst


def _pick_bias(model, inputs, max_words, n_beam, eos_offset=None, tries=200):
    """set the classifier bias to base + BIAS_SIGMA * noise(seed) for the first seed whose eager search has clear
    margins; eos_offset: [SEP]'s bias then sits that far above the largest other bias.  -> the seed"""
    bias = model.decoder.classifier.cls.predictions.bias
    base = bias.detach().clone()
    with torch.no_grad():
        for seed in range(tries):
            g = torch.Generator(device="cuda").manual_seed(1000 + seed)
            b = base + BIAS_SIGMA * torch.randn(base.shape, device="cuda", generator=g)
            if eos_offset is not None:
                b[EOS] = torch.cat([b[:EOS], b[EOS + 1:]]).max() + eos_offset
            bias.copy_(b)
            if _eager_margin(model, *inputs, max_words, n_beam) > 2 * E_STEP:
                print("bias seed %d" % seed)
                return seed
    pytest.fail("no bias among %d seeds gives the eager search margins above 2 E_STEP per step" % tries)


def _inputs(b, seq, vis):
    n = seq.shape[0]
    return seq, vis, b["attention_mask"].view(n, -1), b["video_mask"].view(n, -1)


def _compare(model, inputs, max_words, n_beam):
    hyps, scores = beam_search(model, *inputs, max_words, n_beam=n_beam)
    ghyps, gscores = GraphBeamSearch(model, n_beam=n_beam, max_words=max_words)(*inputs)
    assert ghyps == hyps, (ghyps, hyps)
    worst = max(abs(a - b) / max(len(h), 1) for a, b, h in zip(gscores, scores, hyps))
    print("largest score difference per step %.3e (E_STEP %.1e)" % (worst, E_STEP))
    assert worst <= E_STEP
    return hyps, gscores


def test_rows_do_not_depend_on_other_instances():
    """the assumption that lets finished instances stay in the graph's batch: CachedCaptionDecoder.step's logits of
    the kept instances are the same bits with and without the removed ones"""
    cfg, model, b, seq, vis = _setup(batch_size=4)
    seq, vis, am, vm = _inputs(b, seq, vis)
    n_beam, L = 3, 5
    g = torch.Generator().manual_seed(8)
    tokens = torch.randint(1000, 30522, (seq.shape[0] * n_beam, L), generator=g).cuda()
    keep = [0, 2, 3]
    rows = torch.tensor([i * n_beam + j for i in keep for j in range(n_beam)], device="cuda")
    with torch.no_grad():
        full = CachedCaptionDecoder(model, seq, vis, am, vm, n_beam, L)
        part = CachedCaptionDecoder(model, seq, vis, am, vm, n_beam, L)
        for t in range(L):
            want = full.step(tokens[:, t].contiguous())
            if t == 1:
                part.select(keep)
            got = part.step((tokens[:, t] if t < 1 else tokens[rows, t]).contiguous())
            assert torch.equal(got, want if t < 1 else want[rows]), t


@pytest.mark.parametrize("n_beam,max_words", [(3, 6), (5, 3)])
def test_matches_beam_search(n_beam, max_words):
    cfg, model, b, seq, vis = _setup(batch_size=3)
    inputs = _inputs(b, seq, vis)
    _pick_bias(model, inputs, max_words, n_beam)
    hyps, scores = _compare(model, inputs, max_words, n_beam)
    # the returned score is the hypothesis' log-probability under the full-prefix decoder (teacher forcing)
    with torch.no_grad():
        for i, h in enumerate(hyps):
            ids = torch.tensor([[101] + h[:-1]], device="cuda")
            one = lambda t: t[i:i + 1]
            logits = model.decoder_caption(one(seq), one(vis), one(b["input_ids"]), one(b["attention_mask"]),
                                           one(b["video_mask"]), ids, torch.ones_like(ids), shaped=True,
                                           get_logits=True)[0]
            lp = torch.log_softmax(logits, -1)
            total = float(sum(lp[t, tok] for t, tok in enumerate(h)))
            assert abs(total - scores[i]) <= 0.05 * len(h) + 0.05, (i, total, scores[i])


def test_finished_instances_match_beam_search():
    """[SEP]'s bias swept from far above every other word (all instances finish at step 1) to far below (none finishes
    before the cap), through offsets where instances finish at different steps"""
    cfg, model, b, seq, vis = _setup(batch_size=4)
    inputs = _inputs(b, seq, vis)
    n_beam, max_words = 3, 10
    lengths = {}
    for off in (60.0, -60.0, -1.0, 0.0, 1.0):
        _pick_bias(model, inputs, max_words, n_beam, eos_offset=off)
        hyps, _ = _compare(model, inputs, max_words, n_beam)
        lengths[off] = [len(h) for h in hyps]
        for h in hyps:
            assert EOS not in h[:-1]
            assert h[-1] == EOS or len(h) == max_words
    assert lengths[60.0] == [1] * 4
    assert lengths[-60.0] == [max_words] * 4
    assert any(len(set(lengths[o])) > 1 for o in (-1.0, 0.0, 1.0)), lengths


def test_replay_smaller_batch_and_weight_updates():
    cfg, model, b, seq, vis = _setup(batch_size=4)
    n_beam, max_words = 3, 10
    a = _inputs(b, seq, vis)
    flip = tuple(t.flip(0).contiguous() for t in a)
    small = tuple(t[:3].contiguous() for t in a)
    fresh = lambda x: GraphBeamSearch(model, n_beam=n_beam, max_words=max_words)(*x)
    search = GraphBeamSearch(model, n_beam=n_beam, max_words=max_words)
    first = search(*a)
    assert first == fresh(a)
    assert search(*flip) == fresh(flip)          # a second batch of the same shape replays the same graphs
    assert search(*small) == fresh(small)        # a smaller last batch gets graphs of its own
    assert search(*a) == first
    # an optimizer step updates the parameters in place: the arena is refreshed and the graphs read the new weights
    params = [p for p in model.decoder.parameters() if p.requires_grad]
    g = torch.Generator(device="cuda").manual_seed(2)
    for p in params:
        p.grad = torch.randn(p.shape, device="cuda", generator=g)
    torch.optim.SGD(params, lr=0.05).step()
    for p in params:
        p.grad = None
    updated = search(*a)
    assert updated == fresh(a)
    assert updated[1] != first[1]
    # a parameter the graphs read in place (a LayerNorm weight) moves to new memory: the searcher captures again
    w = model.decoder.decoder.layer[0].output.LayerNorm.weight
    with torch.no_grad():
        w.data = w.data.clone()
        w.mul_(0.5)
    moved = search(*a)
    assert moved == fresh(a)
    assert moved[1] != updated[1]


def test_training_mode_raises():
    cfg, model, b, seq, vis = _setup(batch_size=2)
    search = GraphBeamSearch(model, n_beam=2, max_words=4)
    model.train()
    with pytest.raises(RuntimeError, match="eval"):
        search(*_inputs(b, seq, vis))
