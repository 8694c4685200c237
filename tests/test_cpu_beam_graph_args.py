"""CPU: the argument checks of GraphBeamSearch (univl_b200/caption.py) and of the beam entry points of the C ABI, which
reject bad input before touching a device."""
import types

import pytest
import torch

from univl_b200 import lib, ops
from univl_b200.caption import GraphBeamSearch

H = 768


def _fake_model(positions=16, cross_positions=64):
    emb = types.SimpleNamespace(word_embeddings=types.SimpleNamespace(weight=torch.zeros(50, H)),
                                position_embeddings=types.SimpleNamespace(weight=torch.zeros(positions, H)))
    cross = types.SimpleNamespace(embeddings=types.SimpleNamespace(
        position_embeddings=types.SimpleNamespace(weight=torch.zeros(cross_positions, H))))
    return types.SimpleNamespace(training=False, decoder=types.SimpleNamespace(embeddings=emb), cross=cross)


@pytest.mark.parametrize("n_beam", [0, 9, -1])
def test_n_beam_outside_one_to_eight(n_beam):
    with pytest.raises(ValueError, match="n_beam"):
        GraphBeamSearch(_fake_model(), n_beam=n_beam, max_words=4)


@pytest.mark.parametrize("max_words", [0, 17])
def test_max_words_beyond_the_position_table(max_words):
    with pytest.raises(ValueError, match="max_words"):
        GraphBeamSearch(_fake_model(positions=16), n_beam=2, max_words=max_words)


def test_limits_are_accepted():
    GraphBeamSearch(_fake_model(positions=16), n_beam=1, max_words=16)
    GraphBeamSearch(_fake_model(positions=16), n_beam=8, max_words=1)


def _args(n=2, W=5, F=7, h=H, am_w=None, vm_f=None):
    return (torch.zeros(n, W, h), torch.zeros(n, F, h), torch.ones(n, W if am_w is None else am_w, dtype=torch.long),
            torch.ones(n, F if vm_f is None else vm_f, dtype=torch.long))


@pytest.mark.parametrize("kw,what", [(dict(h=512), "hidden"), (dict(am_w=6), "input_mask"), (dict(vm_f=3), "mask"),
                                     (dict(W=40, F=30), "cross")])
def test_mismatched_inputs(kw, what):
    search = GraphBeamSearch(_fake_model(), n_beam=2, max_words=4)
    with pytest.raises(ValueError, match=what):
        search(*_args(**kw))


def test_instance_counts_must_agree():
    search = GraphBeamSearch(_fake_model(), n_beam=2, max_words=4)
    seq, vis, am, vm = _args()
    with pytest.raises(ValueError):
        search(seq, vis[:1], am, vm)


def test_training_model_is_refused():
    model = _fake_model()
    search = GraphBeamSearch(model, n_beam=2, max_words=4)
    model.training = True
    with pytest.raises(RuntimeError, match="eval"):
        search(*_args())


@pytest.mark.parametrize("n_beam", [0, 9])
def test_c_abi_rejects_n_beam(n_beam):
    assert lib.load().univl_vocab_beam_topk_workspace(4, n_beam, 1000) < 0
    with pytest.raises(RuntimeError, match="n_beam"):
        lib.call("univl_vocab_beam_topk", 16, 768, 16, 768, None, 16, 16, 4, n_beam, 1000, 768, 16, 16, 16, 16,
                 1 << 20, None)
    with pytest.raises(RuntimeError, match="n_beam"):
        lib.call("univl_beam_advance", 16, 16, 4, n_beam, 1000, 0, 4, 102, 16, 16, 16, 16, 16, 16, 32, None)


def test_c_abi_rejects_bad_steps():
    with pytest.raises(RuntimeError, match="max_words"):
        lib.call("univl_beam_advance", 16, 16, 4, 2, 1000, 4, 4, 102, 16, 16, 16, 16, 16, 16, 32, None)
    with pytest.raises(RuntimeError, match="anc_in == anc_out"):
        lib.call("univl_beam_advance", 16, 16, 4, 2, 1000, 0, 4, 102, 16, 16, 16, 16, 16, 16, 16, None)
    with pytest.raises(RuntimeError, match="n_beam <= V"):
        lib.call("univl_vocab_beam_topk", 16, 768, 16, 768, None, 16, 16, 4, 5, 4, 768, 16, 16, 16, 16, 1 << 20, None)


def test_ops_wrapper_rejects_n_beam():
    x = torch.zeros(10, 768, dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="n_beam"):
        ops.vocab_beam_topk(x, x, None, None, None, 9)
    with pytest.raises(ValueError, match="n_beam"):
        ops.vocab_beam_topk(x, x, None, None, None, 3)      # 3 does not divide 10 rows
