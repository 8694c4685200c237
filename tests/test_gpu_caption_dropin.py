"""GPU: the reference's caption evaluation (main_task_caption.eval_epoch, unmodified, from oracle/_ref) through
`univl_b200.launcher`, with UNIVL_DECODE_CACHE off and prefix: the same hyp.txt.

Under prefix the launcher loads univl_b200.modules.beam as `modules.beam`, so the driver runs the host Beam on CUDA
tensors and decoder_caption runs incrementally (a spy on the decode kernel shows it).  The default path takes int64
masks only, so the switch-off run casts the driver's uint8 decoder mask; the prefix run gets it as the driver builds it.

Why equal captions follow from the logit tolerance and are not luck: the classifier bias favours one token clearly,
so at every step the best candidate extends the previous best hypothesis (the one hyp.txt reports) and leads the
runner-up by more than 4 s tol, s the step and tol the logit tolerance of tests/test_gpu_caption.py: each of the two
candidate scores is a sum of s log-probabilities, each of which moves by at most 2 tol when the logits move by tol.  No
other candidate can then overtake the best one in the other run, whatever the beams' lower ranks hold, so both runs
report the same best hypothesis.  (With a context-independent bias the n_bm-th and (n_bm + 1)-th candidates are often
two orders of the same tokens, with equal bias sums, so that margin cannot be made decisive; hyp.txt does not depend on
it.)"""
import argparse
import importlib
import importlib.util
import os
import sys

import pytest
import torch

from oracle import build_ref, synth
from tests.model_util import build_model
from univl_b200 import ops

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAP = 5          # decoding steps (the driver's --max_words loop bound)
FAVOURED = 1000  # the token the classifier bias favours


def _bench():
    spec = importlib.util.spec_from_file_location("_bench_caption_eval",
                                                  os.path.join(ROOT, "scripts", "bench_caption_eval.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_reference_caption_eval_gives_the_same_captions_with_the_decode_cache(tmp_path, monkeypatch):
    root = build_ref.ref_root()
    if root is None:
        pytest.skip("reference checkout not staged (oracle/build_ref.py)")
    bench = _bench()
    monkeypatch.setenv("MASTER_PORT", str(29800 + (os.getpid() % 150)))
    monkeypatch.setenv("UNIVL_DECODE_CACHE", "prefix")
    sys.modules.pop("main_task_caption", None)
    drv, checkout_beam = bench.load_driver(root, str(tmp_path))
    try:
        import modules.beam
        from univl_b200.modules import beam as host_beam
        assert modules.beam is host_beam and drv.Beam is host_beam.Beam   # the launcher's swap under the switch

        cfg = synth.task_config(mode="caption", batch_size=3, text_layers=2, visual_layers=1, cross_layers=1,
                                decoder_layers=2, max_words=16, max_frames=12)
        model = build_model(cfg, seed=0)
        model.eval()
        pred = model.decoder.classifier.cls.predictions
        with torch.no_grad():
            pred.transform.LayerNorm.weight.mul_(0.1)                 # the model's own logits: about +-0.5
            pred.bias[FAVOURED] = 30.0
            pred.bias[FAVOURED + 1:FAVOURED + 5] = torch.tensor([15.0, 14.0, 13.0, 12.0])
        loader = bench.make_loader(cfg, 6, 3, seed=9)                  # two batches of three instances

        calls = {"decode": 0, "scale": 0.0}
        real_decode = ops.attention_decode_fwd

        def decode(*a, **k):
            calls["decode"] += 1
            return real_decode(*a, **k)
        monkeypatch.setattr(ops, "attention_decode_fwd", decode)
        real_caption = model.decoder_caption
        margins = []

        class Recorded(checkout_beam):
            """the checkout's Beam, recording each step's lead of the best candidate and its parent"""

            def advance(self, word_prob, word_length=None):
                lk = word_prob + self.scores.unsqueeze(1) if self.prev_ks else word_prob[0]
                top = lk.reshape(-1).topk(2).values
                done = super(Recorded, self).advance(word_prob, word_length)
                margins.append((len(self.prev_ks), float(top[0] - top[1]), int(self.prev_ks[-1][0])))
                return done

        def run(mode, beam, cast):
            monkeypatch.setenv("UNIVL_DECODE_CACHE", mode)
            drv.Beam = beam

            def caption(*a, **k):
                a = a[:6] + (a[6].long(),) + a[7:] if cast else a
                out = real_caption(*a, **k)
                calls["scale"] = max(calls["scale"], float(out.abs().max()))
                return out
            model.decoder_caption = caption
            out_dir = tmp_path / mode
            out_dir.mkdir()
            nlg = bench.FakeNLGEval()
            args = argparse.Namespace(max_words=CAP, output_dir=str(out_dir), datatype="youcook")
            try:
                drv.eval_epoch(args, model, loader, bench.FakeTokenizer(), torch.device("cuda", 0), 1, nlgEvalObj=nlg)
            finally:
                del model.decoder_caption
            return (out_dir / "hyp.txt").read_text(), nlg.calls[-1][1]

        off_txt, off_hyps = run("off", Recorded, cast=True)
        assert calls["decode"] == 0
        on_txt, on_hyps = run("prefix", host_beam.Beam, cast=False)
        assert calls["decode"] > 0                                      # the incremental path ran
        assert on_txt == off_txt and on_hyps == off_hyps
        assert len(off_hyps) == 6 and all(h.split() == ["w%d" % FAVOURED] * CAP for h in off_hyps)
        tol = 2.0 ** -6 * max(calls["scale"], 1.0) + 2e-2
        assert len(margins) == 6 * CAP
        for step, lead, parent in margins:
            assert parent == 0 or step == 1, (step, parent)             # the best extends the previous best
            assert lead > 4 * step * tol, (step, lead, tol)
    finally:
        if torch.distributed.is_initialized():
            torch.distributed.destroy_process_group()
        sys.modules.pop("main_task_caption", None)
