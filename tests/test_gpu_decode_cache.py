"""GPU: `UniVL.decoder_caption` under UNIVL_DECODE_CACHE=prefix (caption.PrefixDecodeCache) against the full-prefix
path, on call sequences shaped like the caption driver's beam search (main_task_caption.py:434-517): every row's
prefix grows by one token per call, beams reorder, finished instances leave.  The full [R, t, vocab] logits are
compared under the cached decoder's tolerance (tests/test_gpu_caption.py); a spy on the decode kernel shows which
calls ran incrementally, one on `_get_decoder_score` which ran the full path."""
import pytest
import torch

from oracle import synth
from tests.model_util import build_model, to_device
from univl_b200 import ops

pytestmark = pytest.mark.gpu


def _setup(W, F, ragged, batch_size=3):
    cfg = synth.task_config(mode="caption", batch_size=batch_size, text_layers=2, visual_layers=1, cross_layers=1,
                            decoder_layers=2, max_words=W, max_frames=F)
    batch = to_device(synth.make_batch(cfg, seed=31, ragged=ragged))
    model = build_model(cfg, seed=0)
    model.eval()
    with torch.no_grad():
        seq, vis = model.get_sequence_visual_output(batch["input_ids"], batch["token_type_ids"],
                                                    batch["attention_mask"], batch["video"], batch["video_mask"])
    flat = {k: v.view(-1, *v.shape[2:]) for k, v in batch.items()}
    return model, seq, vis, flat


class Spy:
    def __init__(self, monkeypatch, model):
        self.decode = 0
        self.full = 0
        real_decode, real_full = ops.attention_decode_fwd, model._get_decoder_score

        def decode(*a, **k):
            self.decode += 1
            return real_decode(*a, **k)

        def full(*a, **k):
            self.full += 1
            return real_full(*a, **k)
        monkeypatch.setattr(ops, "attention_decode_fwd", decode)
        monkeypatch.setattr(model, "_get_decoder_score", full)

    def take(self):
        out = (self.decode, self.full)
        self.decode = self.full = 0
        return out


def _close(got, want):
    scale = max(float(want.abs().max()), 1.0)
    err = float((got - want).abs().max())
    assert got.shape == want.shape and got.dtype == want.dtype
    assert err <= 2.0 ** -6 * scale + 2e-2, (err, scale)
    return err / scale


def _call(model, monkeypatch, mode, enc, prefix, mask=None, get_logits=True):
    monkeypatch.setenv("UNIVL_DECODE_CACHE", mode)
    seq, vis, ids, am, vm = enc
    with torch.no_grad():
        return model.decoder_caption(seq, vis, ids, am, vm, prefix, torch.ones_like(prefix) if mask is None else mask,
                                     shaped=True, get_logits=get_logits)


@pytest.mark.parametrize("W,F,ragged", [(16, 16, True), (128, 160, False)], ids=["16x16", "288keys"])
def test_driver_like_calls_match_the_full_path(monkeypatch, W, F, ragged):
    model, seq, vis, b = _setup(W, F, ragged)
    n_inst, n_bm, L = seq.shape[0], 3, 7
    rep = lambda t: t.repeat_interleave(n_bm, 0)     # the driver's repeat(1, n_bm, 1).view(n_inst * n_bm, ...)
    enc = (rep(seq), rep(vis), rep(b["input_ids"]), rep(b["attention_mask"]), rep(b["video_mask"]))
    g = torch.Generator().manual_seed(7)
    prefix = torch.full((n_inst * n_bm, 1), 101, dtype=torch.long, device="cuda")
    spy = Spy(monkeypatch, model)
    active = n_inst
    n_layers = len(model.decoder.decoder.layer)
    for t in range(1, L + 1):
        on = _call(model, monkeypatch, "prefix", enc, prefix)
        decode, full = spy.take()
        assert full == 0 and decode == 2 * n_layers, (t, decode, full)   # incremental on every call
        off = _call(model, monkeypatch, "off", enc, prefix)
        spy.take()
        _close(on, off)
        # next prefix: every beam continues a random hypothesis of its instance (hypothesis 0 at the first step)
        origin = torch.randint(0, n_bm if t > 1 else 1, (active, n_bm), generator=g).cuda()
        rows = (torch.arange(active, device="cuda")[:, None] * n_bm + origin).reshape(-1)
        words = torch.randint(1000, 30522, (active * n_bm, 1), generator=g).cuda()
        prefix = torch.cat([prefix.index_select(0, rows), words], 1)
        if t == 3:   # instance 1 finishes: the driver drops its rows (collate_active_info)
            keep = torch.tensor([i for i in range(active) if i != 1], device="cuda")
            keep_rows = (keep[:, None] * n_bm + torch.arange(n_bm, device="cuda")).reshape(-1)
            enc = tuple(x.index_select(0, keep_rows) for x in enc)
            prefix = prefix.index_select(0, keep_rows)
            active -= 1


def test_calls_that_cannot_continue_take_the_full_path(monkeypatch):
    model, seq, vis, b = _setup(16, 16, True)
    n_inst, n_bm = seq.shape[0], 2
    rep = lambda t: t.repeat_interleave(n_bm, 0)
    enc = (rep(seq), rep(vis), rep(b["input_ids"]), rep(b["attention_mask"]), rep(b["video_mask"]))
    g = torch.Generator().manual_seed(3)
    R = n_inst * n_bm
    tokens = torch.randint(1000, 30522, (R, 8), generator=g).cuda()
    tokens[:, 0] = 101
    spy = Spy(monkeypatch, model)
    n_layers = len(model.decoder.decoder.layer)

    def both(t, enc_=enc, prefix=None, mask=None):
        prefix = tokens[:, :t].contiguous() if prefix is None else prefix
        on = _call(model, monkeypatch, "prefix", enc_, prefix, mask)
        counts = spy.take()
        off = _call(model, monkeypatch, "off", enc_, prefix, mask)
        spy.take()
        return on, off, counts

    for t in (1, 2):
        on, off, counts = both(t)
        assert counts == (2 * n_layers, 0)
        _close(on, off)
    # one flipped bit in one sequence_output row: no parent -> the full path, then a refill of 3 positions
    flipped = enc[0].clone()
    flipped.view(torch.int16).view(-1)[5 * 16 * 768 + 77] ^= 1
    enc_f = (flipped,) + enc[1:]
    on, off, counts = both(3, enc_f)
    assert counts == (3 * 2 * n_layers, 1) and torch.equal(on, off)
    on, off, counts = both(4, enc_f)            # the refilled cache continues
    assert counts == (2 * n_layers, 0)
    _close(on, off)
    # a foreign prefix (an earlier token changed): no parent
    foreign = tokens[:, :5].clone()
    foreign[2, 1] += 1
    on, off, counts = both(5, enc_f, foreign)
    assert counts[1] == 1 and torch.equal(on, off)
    # a zero in decoder_mask, a call with gradients, a training-mode call: the full path, cache untouched
    mask = torch.ones_like(foreign)
    mask[0, -1] = 0
    on, off, counts = both(5, enc_f, foreign, mask)
    assert counts == (0, 1) and torch.equal(on, off)
    off = _call(model, monkeypatch, "off", enc_f, foreign)
    spy.take()
    monkeypatch.setenv("UNIVL_DECODE_CACHE", "prefix")
    with torch.enable_grad():
        on = model.decoder_caption(*enc_f, foreign, torch.ones_like(foreign), shaped=True, get_logits=True)
    assert spy.take() == (0, 1)
    assert torch.equal(on, off)
    model.train()
    assert "_univl_decode_cache" not in model.__dict__          # released on the way back into training mode
    with torch.no_grad():
        on = model.decoder_caption(*enc_f, foreign, torch.ones_like(foreign), shaped=True, get_logits=True)
        monkeypatch.setenv("UNIVL_DECODE_CACHE", "off")
        off = model.decoder_caption(*enc_f, foreign, torch.ones_like(foreign), shaped=True, get_logits=True)
    assert spy.take() == (0, 2) and torch.equal(on, off)
    model.eval()
    # argmax output (get_logits=False) after a fresh fill
    on = _call(model, monkeypatch, "prefix", enc, tokens[:, :1].contiguous(), get_logits=False)
    off = _call(model, monkeypatch, "off", enc, tokens[:, :1].contiguous(), get_logits=True)
    assert on.shape == (R, 1) and on.dtype == torch.long
    top2 = off.topk(2, -1).values
    clear = (top2[..., 0] - top2[..., 1]) > 0.1
    assert torch.equal(on[clear], off.max(-1)[1][clear])
