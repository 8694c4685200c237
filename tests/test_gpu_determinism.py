"""GPU: a retrieval fine-tuning (FT-Align) training step computes the same bits every time it runs.

No cross-CTA floating-point atomic is on this path: split-K weight gradients, LayerNorm / embedding / bias / attention
bias gradients, the similarity head and the optimizer's norms all add partial rows in a fixed order.  (The other
training modes' softmax cross-entropy sums its rows in row order too; the one float atomic left on a training path is
MIL-NCE's dsim, whose cells each take at most two addends onto zero, which commute.)  So two identical
models and optimizers fed the same batch agree bit for bit in the loss, every gradient, every parameter and the Adam
moments — with or without SMs reserved for a concurrent collective, and between an eager step and a CUDA-graph replay
of it.  bench.py's --dump-outputs files, the README's statement of that claim, are compared byte for byte."""
import os
import subprocess
import sys

import pytest
import torch

from oracle import synth
from tests.model_util import build_model, to_device
from univl_b200 import runtime as rt

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = 1234


def _cfg():
    return synth.task_config(mode="ft_align", batch_size=6, text_layers=2, visual_layers=1, cross_layers=2,
                             max_words=16, max_frames=12)


def _model_and_opt(cfg, sd):
    """the model and the driver's optimizer; torch.manual_seed first: the dropout seed is torch.initial_seed()"""
    from univl_b200.optim import FusedBertAdam
    torch.manual_seed(SEED)
    model = build_model(cfg, sd=sd, dropout=0.1)
    named = list(model.named_parameters())
    no_decay = ["bias", "LayerNorm.bias", "LayerNorm.weight"]
    groups = [{"params": [p for n, p in named if not any(nd in n for nd in no_decay)], "weight_decay": 0.01},
              {"params": [p for n, p in named if any(nd in n for nd in no_decay)], "weight_decay": 0.0}]
    opt = FusedBertAdam(groups, lr=1e-4, warmup=0.1, t_total=100, max_grad_norm=1.0, global_clip_norm=1.0,
                        model=model)
    opt._build()
    return model, opt


def _step(model, opt, batch, reserve=0):
    opt.zero_grad()
    loss = model(**batch)
    rt.reserve_sms(reserve)             # as bench.py does around backward phases that share the GPU with an all-reduce
    try:
        loss.backward()
    finally:
        rt.reserve_sms(0)
    opt.step()
    return loss


def _state(loss, opt):
    torch.cuda.synchronize()
    return {"loss": loss.detach().clone(), "grads": opt.g.clone(), "params": opt.p.clone(), "m": opt.m.clone(),
            "v": opt.v.clone()}


def _assert_same(a, b, what):
    for k in a:
        assert torch.equal(a[k], b[k]), "%s: %s differs" % (what, k)


def test_training_step_twice_gives_identical_bits():
    cfg = _cfg()
    sd = synth.make_state_dict(cfg, seed=2)
    batch = to_device(synth.make_batch(cfg, seed=3))
    runs = []
    for reserve in (0, 0, 40):
        model, opt = _model_and_opt(cfg, sd)
        states = []
        for _ in range(2):
            states.append(_state(_step(model, opt, batch, reserve), opt))
        runs.append(states)
        del model, opt
    assert float(runs[0][0]["grads"].abs().max()) > 0
    assert not torch.equal(runs[0][0]["params"], runs[0][1]["params"])     # the steps did something
    for r, what in ((1, "second model"), (2, "40 SMs reserved in backward")):
        for s in range(2):
            _assert_same(runs[0][s], runs[r][s], "%s, step %d" % (what, s + 1))


def test_graph_replay_matches_eager_step_bitwise():
    """one eager step and one CUDA-graph replay of the same step, each from the same parameters, optimizer state and
    device RNG {seed, epoch}"""
    cfg = _cfg()
    sd = synth.make_state_dict(cfg, seed=4)
    batch = to_device(synth.make_batch(cfg, seed=5))
    model, opt = _model_and_opt(cfg, sd)
    arena = opt.flat.arena
    rng0 = torch.tensor([SEED, 7], dtype=torch.int64, device="cuda")
    # warm up on a side stream (allocator pools, lazy initialisation) before capturing
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            _step(model, opt, batch)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    keep = {k: t.clone() for k, t in (("p", opt.p), ("m", opt.m), ("v", opt.v), ("shadow", opt.shadow),
                                      ("step", opt.step_dev))}

    def restore():
        opt.p.copy_(keep["p"])
        opt.m.copy_(keep["m"])
        opt.v.copy_(keep["v"])
        opt.shadow.copy_(keep["shadow"])
        opt.step_dev.copy_(keep["step"])
        arena.rng_state.copy_(rng0)
        arena.fresh = True

    restore()
    eager = _state(_step(model, opt, batch), opt)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static_loss = _step(model, opt, batch)
    restore()
    graph.replay()
    replay = _state(static_loss, opt)
    assert int(arena.rng_state[1]) == 8                                     # one epoch advance inside the step
    _assert_same(eager, replay, "graph replay vs eager")


def test_bench_dump_outputs_identical_across_runs(tmp_path):
    """two runs of `bench.py --dump-outputs` with the same arguments write byte-identical files"""
    dirs = []
    for i in range(2):
        d = tmp_path / ("run%d" % i)
        cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", "1", "--warmup", "1",
               "--no_cpu_baseline", "--no_e2e", "--profile_steps", "0", "--dump-outputs", str(d)]
        r = subprocess.run(cmd, cwd=str(tmp_path), capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stderr[-4000:]
        dirs.append(d)
    names = sorted(os.listdir(dirs[0]))
    assert names == sorted(os.listdir(dirs[1])) and "loss.npy" in names and "grads_sample.npy" in names
    for n in names:
        assert (dirs[0] / n).read_bytes() == (dirs[1] / n).read_bytes(), n
