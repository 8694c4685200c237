"""Beam search state of the caption driver (main_task_caption.py:434-517), with the hypotheses kept on the host.

The surface and the arithmetic of the reference's `modules.beam.Beam`: the score add and the top-k over beam x vocabulary
run on the device tensors as there, and the beam finishes when its top hypothesis ends in [SEP].  The difference is
where the bookkeeping lives: each `advance` copies its n_bm scores and ids to the host in ONE transfer, and the
back-pointers are walked over host lists, so `get_current_state` (called once per instance per decoding step) reads
nothing from the device.  `launcher.install_shadow` loads this module as `modules.beam` under UNIVL_DECODE_CACHE=prefix.
"""
import torch


class Constants(object):
    """ids of the special tokens: [PAD] 0, [UNK] 1, [CLS] 2, [SEP] 3 unless a tokenizer's vocabulary gives them"""

    PAD_WORD, UNK_WORD, BOS_WORD, EOS_WORD = "[PAD]", "[UNK]", "[CLS]", "[SEP]"

    def __init__(self):
        self.PAD, self.UNK, self.BOS, self.EOS = 0, 1, 2, 3

    @classmethod
    def from_tokenizer(cls, tokenizer):
        c = cls()
        c.PAD, c.UNK = tokenizer.vocab[c.PAD_WORD], tokenizer.vocab[c.UNK_WORD]
        c.BOS, c.EOS = tokenizer.vocab[c.BOS_WORD], tokenizer.vocab[c.EOS_WORD]
        return c


class Beam(object):
    """`size` hypotheses of one instance.  scores / all_scores are device tensors (the running sums the next advance
    adds to); prev_ks / next_ys are host LongTensors, one per step (next_ys starts with [CLS] for every hypothesis)."""

    def __init__(self, size, device=False, tokenizer=None):
        self.constants = Constants() if tokenizer is None else Constants.from_tokenizer(tokenizer)
        self.size = size
        self._done = False
        self.scores = torch.zeros((size,), dtype=torch.float, device=device)
        self.all_scores = []
        self.prev_ks = []
        self.next_ys = [torch.full((size,), self.constants.BOS, dtype=torch.long)]
        self._host_scores = torch.zeros((size,), dtype=torch.float)
        self._ks = []                                  # host lists behind prev_ks / next_ys
        self._ys = [[self.constants.BOS] * size]

    @property
    def done(self):
        return self._done

    def advance(self, word_prob, word_length=None):
        """word_prob [size, vocab] log-probabilities of every hypothesis' next word -> True once finished"""
        num_words = word_prob.size(1)
        if self.prev_ks:
            beam_lk = word_prob + self.scores.unsqueeze(1).expand_as(word_prob)
        else:
            beam_lk = word_prob[0]                     # the hypotheses are identical at the first step
        best_scores, best_ids = beam_lk.view(-1).topk(self.size, 0, True, True)
        self.all_scores.append(self.scores)
        self.scores = best_scores
        # fp32 scores and ids below 2^53 are exact in fp64: one transfer carries both
        host = torch.stack([best_scores.double(), best_ids.double()]).cpu()
        self._host_scores = host[0].float()
        ids = host[1].long()
        prev_k = ids // num_words
        word = ids - prev_k * num_words
        self.prev_ks.append(prev_k)
        self.next_ys.append(word)
        self._ks.append(prev_k.tolist())
        self._ys.append(word.tolist())
        if self._ys[-1][0] == self.constants.EOS:
            self._done = True
        return self._done

    def sort_scores(self):
        """(scores, hypothesis indices), best first (host tensors).  The sort is stable: hypotheses with exactly equal
        scores keep their top-k order, where the reference's unstable device sort may order them either way."""
        return torch.sort(self._host_scores, dim=0, descending=True, stable=True)

    def get_the_best_score_and_idx(self):
        scores, ids = self.sort_scores()
        return scores[1], ids[1]

    def get_current_state(self):
        return self.get_tentative_hypothesis()

    def get_current_origin(self):
        return self.prev_ks[-1]

    def get_tentative_hypothesis(self):
        """LongTensor [size, steps + 1]: every hypothesis from [CLS], best first"""
        if len(self._ys) == 1:
            return self.next_ys[0].unsqueeze(1)
        _, keys = self.sort_scores()
        return torch.LongTensor([[self.constants.BOS] + self.get_hypothesis(k) for k in keys.tolist()])

    def get_hypothesis(self, k):
        """the words of hypothesis k (without [CLS]), walked back through the back-pointers"""
        k = int(k)
        hyp = []
        for j in range(len(self._ks) - 1, -1, -1):
            hyp.append(self._ys[j + 1][k])
            k = self._ks[j][k]
        return hyp[::-1]
