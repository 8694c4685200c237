"""GPU: univl_b200.ddp.PhasedBackward — cutting the backward at text-encoder layers (so the gradient exchange of one
phase can overlap the next, the role of DDP's bucket hooks in main_task_retrieval.py:197-198) must leave exactly the
gradients of the single `loss.backward()`, and the per-phase ranges must tile the flat gradient buffer."""
import pytest
import torch

from oracle import synth
from tests.model_util import build_model, to_device

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("mode,cuts", [("ft_align", (1,)), ("caption", (2, 1)), ("pretrain2", (1,))])
def test_phases_reproduce_single_backward(mode, cuts):
    from univl_b200 import optim
    from univl_b200.ddp import PhasedBackward
    kw = dict(mode=mode, batch_size=4, max_words=16, max_frames=16, text_layers=3, visual_layers=1, cross_layers=1,
              decoder_layers=1)
    cfg = synth.task_config(**kw)
    sd = synth.make_state_dict(cfg, seed=3)
    batch = to_device(synth.make_batch(cfg, seed=5))

    def flat_grads(phased_cuts):
        model = build_model(cfg, sd=sd)             # dropout 0: both runs see the same function
        flat = optim.flatten(model)
        flat.zero_grad()
        ph = PhasedBackward(model, flat, phased_cuts) if phased_cuts else None
        if ph:
            ph.begin()
        loss = model(**batch)
        if ph:
            done = torch.zeros_like(flat.g, dtype=torch.bool)
            released = {}
            for i in range(ph.n_phases):
                ph.backward(i, loss if i == 0 else None)
                torch.cuda.synchronize()
                snap = flat.g.clone()
                for a, b in ph.ranges[i]:
                    assert not done[a:b].any()
                    done[a:b] = True
                if i:   # ranges released by earlier phases must not change afterwards
                    for j in range(i):
                        for a, b in ph.ranges[j]:
                            assert torch.equal(snap[a:b], released[j][(a, b)]), (i, j, a, b)
                released[i] = {(a, b): snap[a:b].clone() for a, b in ph.ranges[i]}
            assert bool(done.all()) and ph.covered() == flat.total
        else:
            loss.backward()
        torch.cuda.synchronize()
        return float(loss.detach()), flat.g.clone()

    l0, g0 = flat_grads(None)
    l1, g1 = flat_grads(cuts)
    assert float(g0.norm()) > 0
    # same kernels on the same inputs, and every gradient sum is added in a fixed order: the same bits
    assert torch.equal(g1, g0)
    assert l0 == l1
