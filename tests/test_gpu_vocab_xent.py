"""GPU: the fused vocabulary cross-entropy (UNIVL_VOCAB_LOSS=fused: univl_vocab_xent_fwd / _bwd, csrc/gemm_wgmma.cu),
which computes CrossEntropy(x W^T + bias, labels, ignore_index=-1) without writing the logits.

Written bounds (U = 2^-24, the fp32 unit roundoff; the constants are tests/gemm_check.py's):
  logit    eL = C_ACC K U |x||W|^T + EPI_ROUND (|x||W|^T + |bias|): the wgmma accumulation and the bias add.
  lse      |d lse| <= max_c eL (lse moves by at most its largest argument's error)
           + (33 ct + 3 chunks + 8) U: the longest chain of fp32 adds and rescalings of the exp sum (a thread adds 32
             columns and rescales once per 128-column tile of its chunk of ct tiles, then two quad folds and the chunk
             fold), each a relative U on a sum of positive terms
           + 2 MUFU + 2 U range: ex2 / lg2 approximation and the rounding of the exponent argument (range = the row's
             max - min logit) + 2 U |lse|.
  loss     per row B_lse + eL[label] + U |nll|, summed over a group with (R / 512 + 12) U sum |nll| for the fixed-order
           sum, divided by the count, averaged over groups with (G + 2) 2 U |loss|.
  dl       g E (eL + B_lse + MUFU + U |l - lse|) + (BF16_ROUND + 4 U) |dl| with E = exp(l - lse), g = (1 / G) / count:
           the logit and lse errors move E by E times their sum; then the fp32 arithmetic and the bf16 store.
  dx, dW, db   the dl bound carried through the existing GEMMs / colsum (|B_dl| |W|, |B_dl|^T |x|, sum B_dl) plus their
           own accumulation terms (gemm_check.elem_bound's) and the bf16 store of dx.
test_checker_rejects_a_dropped_chunk_and_a_wrong_label shows these bounds still reject one vocabulary chunk missing
from the lse and a label logit read from the wrong column."""

import pytest
import torch

from tests.gemm_check import BF16_ROUND, C_ACC, EPI_ROUND, U, within
from tests.test_cpu_vocab_xent_args import vx_chunks
from univl_b200 import ops
from univl_b200 import runtime as rt

pytestmark = pytest.mark.gpu

DEV = "cuda"
BF16 = torch.bfloat16
K = 768
MUFU = 2.0 ** -21  # ex2.approx / lg2.approx: about 2^-22 relative (lg2: absolute); twice that


class _Head(torch.nn.Module):
    """a tied vocabulary projection: W fp32 [V, K] (its bf16 arena copy is the GEMM operand) and bias [V]"""

    def __init__(self, V, seed):
        super().__init__()
        g = torch.Generator(device=DEV).manual_seed(seed)
        self.weight = torch.nn.Parameter(0.05 * torch.randn(V, K, device=DEV, generator=g))
        self.bias = torch.nn.Parameter(torch.randn(V, device=DEV, generator=g))


def _inputs(T, V, G, seed, empty_group=None):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(T, K, device=DEV, generator=g).to(BF16)
    labels = torch.randint(0, V, (T,), device=DEV, generator=g)
    labels[torch.rand(T, device=DEV, generator=g) < 0.3] = -1  # ragged: about 30 % unscored
    R = T // G
    labels[::R] = torch.randint(0, V, (G,), device=DEV, generator=g)  # every group scores a row ...
    if empty_group is not None:
        labels[empty_group * R:(empty_group + 1) * R] = -1             # ... but this one
    return x, labels


def _ctx(head):
    return rt.use_model(head, torch.device("cuda", torch.cuda.current_device()))


def _step(head, x, labels, G, mode, monkeypatch):
    """loss, dx, dW, db of one ProjXentFn forward + backward under UNIVL_VOCAB_LOSS=mode"""
    monkeypatch.setenv("UNIVL_VOCAB_LOSS", mode)
    head.weight.grad = head.bias.grad = None
    with _ctx(head):
        xr = x.clone().requires_grad_()
        loss = ops.ProjXentFn.apply(xr, head.weight, head.bias, labels, None, 0, True, False, G)
        loss.backward()
    torch.cuda.synchronize()
    return loss.detach(), xr.grad, head.weight.grad.clone(), head.bias.grad.clone()


def _w16(head):
    with _ctx(head) as arena:
        return arena.bf16(head.weight)


def _fused(w16, bias, x, labels, G):
    loss, lse, sc = ops.vocab_xent_fwd(x, w16, bias, labels, G)
    dl = ops.vocab_xent_bwd(x, w16, bias, labels, lse, sc, None, G)
    return loss, lse, sc, dl


def _raw(head, x, labels, G):
    """(loss, lse, sum_count, dl) of the raw fused entry points, upstream gradient 1"""
    return _fused(_w16(head), head.bias.detach(), x, labels, G)


def _raw_logits_mode(head, x, labels, G):
    """(loss, lse, dl) of today's path: fp32 logits, univl_softmax_xent_fwd / _bwd"""
    with _ctx(head) as arena:
        w16 = arena.bf16(head.weight)
        T, V = x.shape[0], w16.shape[0]
        ld = ops._ld_pad(V)
        logits = torch.empty((T, ld), dtype=torch.float32, device=DEV)[:, :V]
        ops.gemm(x, w16, T, V, K, logits, epi=ops.EPI_F32, bias=head.bias)
        lse = torch.empty(T, device=DEV)
        sc = torch.empty(2 * G, device=DEV)
        loss = torch.empty((), device=DEV)
        rt.call("univl_softmax_xent_fwd", logits.data_ptr(), logits.stride(0), labels.data_ptr(), None,
                lse.data_ptr(), sc.data_ptr(), loss.data_ptr(), T, V, 0, -1, G)
        dl = torch.empty((T, ld), dtype=BF16, device=DEV)
        rt.call("univl_softmax_xent_bwd", logits.data_ptr(), logits.stride(0), labels.data_ptr(), None,
                lse.data_ptr(), sc.data_ptr(), None, dl.data_ptr(), ld, T, V, 0, -1, G)
    return loss, lse, dl


class _Ref:
    """float64 statement of the loss and its gradients, with the bounds of the module docstring"""

    def __init__(self, head, x, labels, G):
        T = x.shape[0]
        V = head.weight.shape[0]
        R = T // G
        x64 = x.double()
        W64 = head.weight.detach().to(BF16).double()
        b64 = head.bias.detach().double()
        l = x64 @ W64.t() + b64
        mag = x64.abs() @ W64.abs().t()
        eL = C_ACC * K * U * mag + EPI_ROUND * (mag + b64.abs())
        del mag
        self.lse = torch.logsumexp(l, 1)
        chunks, ct = vx_chunks(T, V)
        rng = l.max(1).values - l.min(1).values
        self.b_lse = (eL.max(1).values + (33 * ct + 3 * chunks + 8) * U + 2 * MUFU + 2 * U * rng
                      + 2 * U * self.lse.abs())
        scored = labels != -1
        lab = labels.clamp_min(0)
        self.l, self.labels, self.scored, self.chunks, self.ct = l, labels, scored, chunks, ct
        nll = torch.where(scored, self.lse - l.gather(1, lab[:, None])[:, 0], torch.zeros_like(self.lse))
        b_nll = torch.where(scored, self.b_lse + eL.gather(1, lab[:, None])[:, 0] + U * nll.abs(),
                            torch.zeros_like(nll))
        count = scored.view(G, R).sum(1).double()
        self.count = count
        per = nll.view(G, R).sum(1) / count
        self.loss = per.mean()
        b_per = (b_nll.view(G, R).sum(1) + (R / 512 + 12) * U * nll.abs().view(G, R).sum(1)) / count
        self.b_loss = b_per.mean() + (G + 2) * 2 * U * self.loss.abs()
        g = ((1.0 / G) / count).repeat_interleave(R)
        g = torch.where(scored, g, torch.zeros_like(g))
        E = torch.exp(l - self.lse[:, None])
        onehot = torch.zeros_like(l)
        onehot[torch.arange(T, device=DEV), lab] = 1.0
        self.dl = (E - onehot) * g[:, None]
        self.dl[~scored] = 0.0
        self.b_dl = g[:, None] * E * (eL + self.b_lse[:, None] + MUFU + U * (l - self.lse[:, None]).abs()) \
            + (BF16_ROUND + 4 * U) * self.dl.abs()
        self.b_dl[~scored] = 0.0
        del E, onehot, eL
        self.g = g
        a_dl = self.dl.abs() + self.b_dl
        self.dx = self.dl @ W64
        self.b_dx = self.b_dl @ W64.abs() + (C_ACC * V * U + EPI_ROUND) * (a_dl @ W64.abs())
        self.b_dx = self.b_dx + BF16_ROUND * (self.dx.abs() + self.b_dx)
        self.dW = self.dl.t() @ x64
        self.b_dW = self.b_dl.t() @ x64.abs() + (C_ACC * T * U + EPI_ROUND) * (a_dl.t() @ x64.abs())
        self.db = self.dl.sum(0)
        self.b_db = self.b_dl.sum(0) + (T + 2) * U * a_dl.sum(0)


CASES = [(1, 30522, 1), (127, 1000, 1), (127, 257, 1), (4096, 30522, 1), (4096, 1000, 2), (4096, 257, 2),
         (384, 30522, 3), (384, 257, 3)]


@pytest.mark.parametrize("T,V,G", CASES)
def test_fused_against_fp64(T, V, G, monkeypatch):
    head = _Head(V, seed=T + V)
    for empty in ([None] if G == 1 else [None, G - 1]):
        x, labels = _inputs(T, V, G, seed=3 * T + G, empty_group=empty)
        ref = _Ref(head, x, labels, G)
        what = "T=%d V=%d G=%d empty=%s" % (T, V, G, empty)
        loss, lse, sc, dl = _raw(head, x, labels, G)
        torch.cuda.synchronize()
        within(lse, ref.lse.where(ref.scored, torch.zeros_like(ref.lse)), ref.b_lse.where(ref.scored, 0 * ref.b_lse),
               what + " lse")
        assert torch.equal(sc[G:].double(), ref.count), (sc, ref.count)
        if empty is None:
            within(loss.view(1), ref.loss.view(1), ref.b_loss.view(1), what + " loss")
        else:
            assert torch.isnan(loss), "a group without a scored row makes the loss NaN"
        within(dl[:, :V], ref.dl, ref.b_dl, what + " dl")
        assert bool((dl[:, V:] == 0).all()), "padding columns of dl are zero"
        loss2, dx, dW, db = _step(head, x, labels, G, "fused", monkeypatch)
        assert torch.equal(loss2, loss) or (empty is not None and torch.isnan(loss2))
        within(dx, ref.dx, ref.b_dx, what + " dx")
        within(dW, ref.dW, ref.b_dW, what + " dW")
        within(db, ref.db, ref.b_db, what + " db")
        del ref
        torch.cuda.empty_cache()


def test_checker_rejects_a_dropped_chunk_and_a_wrong_label():
    T, V, G = 4096, 30522, 1
    head = _Head(V, seed=1)
    x, labels = _inputs(T, V, G, seed=2)
    ref = _Ref(head, x, labels, G)
    loss, lse, sc, dl = _raw(head, x, labels, G)
    torch.cuda.synchronize()
    lse_ref = ref.lse.where(ref.scored, torch.zeros_like(ref.lse))
    b_lse = ref.b_lse.where(ref.scored, 0 * ref.b_lse)
    within(lse, lse_ref, b_lse, "lse")
    assert ref.chunks > 1
    # a kernel that left the last chunk out of every row's lse
    cols = (ref.chunks - 1) * ref.ct * 128
    dropped = torch.logsumexp(ref.l[:, :cols], 1).where(ref.scored, torch.zeros_like(ref.lse))
    with pytest.raises(AssertionError):
        within(dropped, lse_ref, b_lse, "lse without the last chunk")
    # a kernel that read every label logit one column to the right
    lab = ref.labels.clamp_min(0)
    shifted = (lab + 1) % V
    nll = ref.lse - ref.l.gather(1, shifted[:, None])[:, 0]
    bad_loss = (nll * ref.scored).sum() / ref.count[0]
    with pytest.raises(AssertionError):
        within(bad_loss.view(1), ref.loss.view(1), ref.b_loss.view(1), "loss with a shifted label column")
    # ... or took the one-hot of one row's gradient at the wrong column
    r = int(ref.scored.nonzero()[0])
    bad = ref.dl.clone()
    bad[r, lab[r]] += ref.g[r]
    bad[r, shifted[r]] -= ref.g[r]
    with pytest.raises(AssertionError):
        within(bad, ref.dl, ref.b_dl, "dl with a wrong label column")
    within(dl[:, :V], ref.dl, ref.b_dl, "dl")


@pytest.mark.parametrize("T,G", [(4096, 1), (384, 3)])
def test_agrees_with_logits_mode(T, G, monkeypatch):
    V = 30522
    head = _Head(V, seed=5)
    x, labels = _inputs(T, V, G, seed=6)
    ref = _Ref(head, x, labels, G)
    loss_f, lse_f, _, dl_f = _raw(head, x, labels, G)
    loss_l, lse_l, dl_l = _raw_logits_mode(head, x, labels, G)
    torch.cuda.synchronize()
    # both sum the same fp32 logits in another order: each within the derived bound of the exact value
    assert abs(float(loss_f) - float(loss_l)) <= 2 * float(ref.b_loss), (float(loss_f), float(loss_l))
    d_lse = (lse_f.double() - lse_l.double()).abs()
    assert bool((d_lse <= 2 * ref.b_lse).all())
    # dl: the same logits through the same formula; only the lse differs, so the two agree up to a bf16 rounding of
    # each and the lse difference's effect exp(l - lse) g |d lse|
    E = torch.exp(ref.l - lse_l.double()[:, None])
    bound = 2 * BF16_ROUND * dl_l[:, :V].double().abs() + 1.01 * ref.g[:, None] * E * d_lse[:, None]
    within(dl_f[:, :V], dl_l[:, :V].double(), bound + 1e-30, "dl fused vs logits")
    # where the two lse agree bit for bit, so does every dl element: the logit tiles are the same GEMM
    same = (lse_f == lse_l) & ref.scored
    print("rows with bit-equal lse: %d of %d scored" % (int(same.sum()), int(ref.scored.sum())))
    assert torch.equal(dl_f[same], dl_l[same])
    assert torch.equal(dl_f[~ref.scored], dl_l[~ref.scored])
    # through ProjXentFn: the loss of both modes
    lf = _step(head, x, labels, G, "fused", monkeypatch)[0]
    ll = _step(head, x, labels, G, "logits", monkeypatch)[0]
    assert abs(float(lf) - float(ll)) <= 2 * float(ref.b_loss)


def test_deterministic_repeat_reserved_graph_and_streams():
    T, V, G = 4096, 30522, 2
    head = _Head(V, seed=8)
    x, labels = _inputs(T, V, G, seed=9)
    w16, bias = _w16(head), head.bias.detach()
    base = _fused(w16, bias, x, labels, G)
    torch.cuda.synchronize()

    def same(out, what):
        for a, b in zip(base, out):
            assert torch.equal(a, b) or (a.isnan().all() and b.isnan().all()), what

    same(_fused(w16, bias, x, labels, G), "second launch")
    rt.reserve_sms(40)
    try:
        same(_fused(w16, bias, x, labels, G), "40 SMs reserved")
    finally:
        rt.reserve_sms(0)
    # CUDA-graph capture of forward + backward, replayed
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _fused(w16, bias, x, labels, G)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = _fused(w16, bias, x, labels, G)
    for t in captured:
        t.fill_(0)
    graph.replay()
    torch.cuda.synchronize()
    same(captured, "graph replay")
    # two streams at once
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    s1.wait_stream(torch.cuda.current_stream())
    s2.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s1):
        o1 = _fused(w16, bias, x, labels, G)
    with torch.cuda.stream(s2):
        o2 = _fused(w16, bias, x, labels, G)
    torch.cuda.synchronize()
    same(o1, "stream 1")
    same(o2, "stream 2")


def _saved_shapes(head, x, labels, mode, monkeypatch):
    monkeypatch.setenv("UNIVL_VOCAB_LOSS", mode)
    shapes = []

    def pack(t):
        shapes.append(tuple(t.shape))
        return t

    with _ctx(head), torch.autograd.graph.saved_tensors_hooks(pack, lambda t: t):
        xr = x.clone().requires_grad_()
        loss = ops.ProjXentFn.apply(xr, head.weight, head.bias, labels, None, 0, True, False, 1)
    del loss
    return shapes


def test_autograd_keeps_nothing_of_size_t_by_v(monkeypatch):
    T, V = 4096, 30522
    head = _Head(V, seed=10)
    x, labels = _inputs(T, V, 1, seed=11)
    fused = _saved_shapes(head, x, labels, "fused", monkeypatch)
    print("fused saves", fused)
    assert fused and all(torch.Size(s).numel() < T * V for s in fused), fused
    assert any(torch.Size(s).numel() >= T * V for s in _saved_shapes(head, x, labels, "logits", monkeypatch))


def test_switch_leaves_nce_and_return_logits_on_todays_path(monkeypatch):
    """target_mode 1 and return_logits=True ignore the switch: the same bits under either value"""
    T, V = 256, 1000
    head = _Head(V, seed=12)
    x, labels = _inputs(T, V, 1, seed=13)
    outs = []
    for mode in ("logits", "fused"):
        monkeypatch.setenv("UNIVL_VOCAB_LOSS", mode)
        with _ctx(head):
            loss, logits = ops.ProjXentFn.apply(x, head.weight, head.bias, labels, None, 0, True, True, 1)
            frames = x.clone()
            vm = torch.ones(T, dtype=torch.long, device=DEV)
            nce_labels = torch.arange(T, device=DEV)
            nce = ops.ProjXentFn.apply(x, frames, None, nce_labels, vm, 1, False, False, 1)
        torch.cuda.synchronize()
        outs.append((logits.clone(), nce.clone()))
    assert torch.equal(outs[0][0], outs[1][0])
    assert torch.equal(outs[0][1], outs[1][1]) or abs(float(outs[0][1]) - float(outs[1][1])) <= T * U * abs(
        float(outs[0][1]))
    monkeypatch.setenv("UNIVL_VOCAB_LOSS", "Fused")
    with _ctx(head), pytest.raises(ValueError, match="UNIVL_VOCAB_LOSS"):
        ops.ProjXentFn.apply(x, head.weight, head.bias, labels, None, 0, True, False, 1)


# ---------------------------------------------------------------------------------------------------------
# model level: the MLM head (pretrain stage two) and the caption head under the switch
# ---------------------------------------------------------------------------------------------------------
def _model_step(cfg, sd, batch, G, mode, monkeypatch):
    from tests.model_util import build_model, grads_by_name, to_device
    if mode is None:
        monkeypatch.delenv("UNIVL_VOCAB_LOSS", raising=False)
    else:
        monkeypatch.setenv("UNIVL_VOCAB_LOSS", mode)
    torch.manual_seed(0)
    model = build_model(cfg, sd=sd, dropout=0.0)
    kw = {} if G == 1 else {"micro_batches": G}
    loss = model(**to_device(batch), **kw)
    loss.backward()
    torch.cuda.synchronize()
    return float(loss.detach()), grads_by_name(model)


MODEL_CASES = [("pretrain2", 1, 1), ("pretrain2", 1, 3), ("pretrain2", 3, 1), ("pretrain2", 3, 3), ("caption", 1, 1),
               ("caption", 1, 3)]


@pytest.mark.parametrize("mode,n_pair,G", MODEL_CASES)
def test_model_step_fused_against_oracle(mode, n_pair, G, monkeypatch):
    """Losses and gradients with UNIVL_VOCAB_LOSS=fused against the CPU oracle: within test_gpu_model_parity.py's
    cross-entropy loss bound (2e-3 |loss|) and its per-tensor gradient bound, or no further from the oracle than the
    logits path is; and against the logits path, within fp32 reordering (loss) and a bf16 rounding of dl (gradients).
    The switch unset and set to "logits" give the same loss and gradient bits."""
    from oracle import synth
    from tests.oracle_util import run_oracle
    from tests.test_gpu_micro_batches import _cfg, _window
    cfg = _cfg(mode, n_pair)
    sd = synth.make_state_dict(cfg, seed=7)
    batch, parts = _window(cfg, G, seed=31)
    loss_u, g_u = _model_step(cfg, sd, batch, G, None, monkeypatch)
    loss_l, g_l = _model_step(cfg, sd, batch, G, "logits", monkeypatch)
    loss_f, g_f = _model_step(cfg, sd, batch, G, "fused", monkeypatch)
    assert set(g_u) == set(g_l) == set(g_f)
    for k in g_l:
        assert torch.equal(g_u[k], g_l[k]), k
    assert loss_u == loss_l
    assert abs(loss_f - loss_l) <= 1e-5 * abs(loss_l), (loss_f, loss_l)
    flat_f = torch.cat([g_f[k].flatten() for k in sorted(g_f)]).double()
    flat_l = torch.cat([g_l[k].flatten() for k in sorted(g_l)]).double()
    rel = float((flat_f - flat_l).norm() / flat_l.norm())
    print("fused vs logits: loss %.3e relative, gradients %.3e relative" % (abs(loss_f - loss_l) / abs(loss_l), rel))
    assert rel <= 2.0 ** -8, rel

    oracle = [run_oracle(cfg, p, sd=sd, backward=True) for p in parts]
    o_loss = sum(float(o[0]) for o in oracle) / G
    o_grads = {k: sum(o[2][k] for o in oracle) / G for k in oracle[0][2]}
    tol = 2e-3 * abs(o_loss)
    assert abs(loss_f - o_loss) <= max(tol, 1.5 * abs(loss_l - o_loss)), (loss_f, loss_l, o_loss)
    norms = {k: float(v.double().norm()) for k, v in o_grads.items() if k in g_f}
    floor = 0.05 * max(norms.values())
    bad = []
    for k, n in norms.items():
        err_f = float((g_f[k].double() - o_grads[k].double()).norm())
        err_l = float((g_l[k].double() - o_grads[k].double()).norm())
        if err_f > 0.10 * max(n, floor) and err_f > 1.5 * err_l + 2.0 ** -12 * n:
            bad.append((k, err_f, err_l, n))
    assert not bad, bad[:5]
