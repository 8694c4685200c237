"""GPU: UniVL.forward(micro_batches=G) runs a gradient-accumulation window of G micro-batches as one batch and returns
(1/G) * sum_g L_g, L_g being the loss of micro-batch g alone.

Why the grouped step can match the accumulation loop to fp32 summation order: every forward kernel is row- or
sequence-local, the pairing-group kernels give each micro-batch exactly the sequences, similarity matrix, negatives and
means it has on its own, and the loss gradients enter with the loop's bits ((1/G) * dsim, (g / G) / count).  What
differs is the order of the cross-row parameter-gradient sums (weight GEMMs over all rows at once, LayerNorm / bias /
embedding partials) and the loss value's mean over groups against the loop's running sum of (1/G) L_g.  (Each group's
cross-entropy sum has the bits of its micro-step's: the same rows, thread striding and block reduction.)  The
models here use 64 text tokens and 12 frames: the fused self-attention kernel packs 128 / S sequences into one row
block, and with an even micro-batch every sequence then sits at the same place in its block as in its own micro-step, so
the tests need not assume how a block's sums treat the other sequences' masked-out keys.  (At the stage-I shape, 45-row
micro-batches of 48-token text, sequences do shift within their blocks; scripts/bench_micro_batches.py measures the
flat gradients of the two ways 6e-6 apart there, still fp32 order.)"""
import pytest
import torch

from oracle import synth
from tests.model_util import build_model, grads_by_name, to_device
from tests.oracle_util import run_oracle
from tests.test_gpu_kernels import _bf, _fused_inputs
from tests.test_gpu_model_parity import loss_tolerance
from univl_b200 import ops
from univl_b200 import runtime as rt

pytestmark = pytest.mark.gpu

DEV = "cuda"
U32 = 2.0 ** -24
SEED = 4321


def _cfg(mode, n_pair=1, b=2, max_words=64, max_frames=12):
    return synth.task_config(mode=mode, batch_size=b, n_pair=n_pair, text_layers=2, visual_layers=1, cross_layers=1,
                             decoder_layers=1, max_words=max_words, max_frames=max_frames)


def _window(cfg, G, seed):
    """G micro-batches, each as the reference dataloader emits one, and their concatenation along the batch"""
    parts = [synth.make_batch(cfg, seed=seed + 17 * g) for g in range(G)]
    return {k: torch.cat([p[k] for p in parts], 0) for k in parts[0]}, parts


def _model_and_opt(cfg, sd, dropout):
    from univl_b200.optim import FusedBertAdam
    torch.manual_seed(SEED)
    model = build_model(cfg, sd=sd, dropout=dropout)
    named = list(model.named_parameters())
    no_decay = ["bias", "LayerNorm.bias", "LayerNorm.weight"]
    groups = [{"params": [p for n, p in named if not any(nd in n for nd in no_decay)], "weight_decay": 0.01},
              {"params": [p for n, p in named if any(nd in n for nd in no_decay)], "weight_decay": 0.0}]
    opt = FusedBertAdam(groups, lr=1e-4, warmup=0.1, t_total=100, max_grad_norm=1.0, global_clip_norm=1.0, model=model)
    opt._build()
    return model, opt


def _grouped(model, opt, batch, **kw):
    opt.zero_grad()
    loss = model(**batch, **kw)
    loss.backward()
    torch.cuda.synchronize()
    return loss.detach().clone(), opt.g.clone()


def _loop(model, opt, parts):
    """the reference driver's accumulation: (loss / G).backward() per micro-batch"""
    opt.zero_grad()
    total = torch.zeros((), device=DEV)
    for p in parts:
        loss = model(**p) / len(parts)
        loss.backward()
        total = total + loss.detach()
    torch.cuda.synchronize()
    return total, opt.g.clone()


def _combine_roundings(G):
    """fp32 roundings in which the grouped loss value and the loop's may differ.  Each micro-batch's loss components
    have the same bits either way; only their combination differs.  The grouped step averages each component over G
    groups (G - 1 adds and a division) and adds the <= 5 components; the loop adds the components, divides by G and
    accumulates G terms.  Every term is >= 0, so each side errs by at most G + 6 roundings of |loss|, and the two
    differ by at most twice that."""
    return 2 * (G + 6)


MODES = [("ft_joint", 1, 2), ("ft_joint", 3, 3), ("ft_align", 1, 2), ("ft_align", 1, 3), ("caption", 1, 2),
         ("caption", 1, 3), ("pretrain1", 3, 2), ("pretrain1", 3, 3), ("pretrain2", 1, 2), ("pretrain2", 3, 3)]


@pytest.mark.parametrize("mode,n_pair,G", MODES)
def test_grouped_step_matches_accumulation_loop(mode, n_pair, G):
    cfg = _cfg(mode, n_pair)
    sd = synth.make_state_dict(cfg, seed=7)
    batch, parts = _window(cfg, G, seed=31)
    batch, parts = to_device(batch), [to_device(p) for p in parts]
    model, opt = _model_and_opt(cfg, sd, dropout=0.0)

    # micro_batches=1 is the plain call on one micro-batch: the same loss and gradient bits
    plain_loss, plain_g = _grouped(model, opt, parts[0])
    one_loss, one_g = _grouped(model, opt, parts[0], micro_batches=1)
    assert torch.equal(plain_g, one_g)
    assert torch.equal(plain_loss, one_loss)

    loss, g = _grouped(model, opt, batch, micro_batches=G)
    ref_loss, ref_g = _loop(model, opt, parts)
    tol = (_combine_roundings(G) + 2) * U32 * abs(float(ref_loss))
    assert abs(float(loss) - float(ref_loss)) <= tol, (float(loss), float(ref_loss), tol)
    # parameter gradients: fp32 sums over <= 4096 rows taken in another order.  The relative error of such a sum is
    # O(sqrt(rows) * 2^-24) ~ 4e-6; 2^-12 leaves a 60x margin yet sits 16x below what one bf16 rounding flip in an
    # activation gradient (2^-8 relative) would cause.
    err = float((g - ref_g).double().norm() / ref_g.double().norm())
    assert float(ref_g.abs().max()) > 0
    assert err <= 2.0 ** -12, err


def test_grouped_loss_is_not_the_big_batch_loss():
    """the objective really is per micro-batch: the B x B retrieval loss of the whole window differs"""
    cfg = _cfg("ft_joint")
    batch, _ = _window(cfg, 2, seed=3)
    batch = to_device(batch)
    cfg_big = _cfg("ft_joint", b=4)
    sd = synth.make_state_dict(cfg, seed=7)
    grouped = float(build_model(cfg, sd=sd)(**batch, micro_batches=2).detach())
    whole = float(build_model(cfg_big, sd=sd)(**batch).detach())
    # fp32 summation order moves these losses by ~1e-6 relative; the objectives differ by far more than that
    assert abs(grouped - whole) > 2.0 ** -12 * abs(whole), (grouped, whole)


# ---------------------------------------------------------------------------------------------------------
# against the CPU oracle run per micro-batch and averaged (bounds of test_gpu_model_parity.py)
@pytest.mark.parametrize("mode,n_pair,G", [("ft_joint", 1, 3), ("ft_align", 1, 2), ("pretrain2", 3, 2)])
def test_grouped_step_matches_oracle_per_micro_batch(mode, n_pair, G):
    cfg = _cfg(mode, n_pair, max_words=24, max_frames=16)
    sd = synth.make_state_dict(cfg, seed=3)
    batch, parts = _window(cfg, G, seed=11)
    model = build_model(cfg, sd=sd)
    loss = model(**to_device(batch), micro_batches=G)
    loss.backward()
    torch.cuda.synchronize()
    grads = grads_by_name(model)

    o_losses, o_grads, tols = [], {}, []
    for p in parts:
        o_loss, o_parts, og = run_oracle(cfg, p, sd=sd, backward=True)
        o_losses.append(float(o_loss))
        for k, v in og.items():
            o_grads[k] = o_grads.get(k, 0) + v.double() / G
        sims = [o_parts["sim_matrix"].detach()]
        if mode == "pretrain2":
            # the joint (mean-pool, MIL-NCE) similarity of this micro-batch: its largest logit scales the NCE bound
            with torch.no_grad():
                d = to_device(p)
                model.eval()
                s, v = model.get_sequence_visual_output(d["input_ids"], d["token_type_ids"], d["attention_mask"],
                                                        d["video"], d["video_mask"])
                sims = [model.get_similarity_logits(s, v, d["attention_mask"], d["video_mask"],
                                                    _pretrain_joint=True).float().cpu()]
                model.train()
        gold = {"loss": float(o_loss), "sim_matrices": sims, "weight_kwargs": {}}
        tols.append(loss_tolerance(cfg, gold, {k: float(v) for k, v in o_parts.items() if k == "mfm_loss"}))
    ref = sum(o_losses) / G
    tol = sum(tols) / G
    assert abs(float(loss) - ref) <= tol, (float(loss), ref, tol)

    assert set(grads) == set(o_grads), sorted(set(grads) ^ set(o_grads))[:8]
    biggest = max(float(v.norm()) for v in o_grads.values())
    floor = 0.05 * biggest
    bad, emu = [], None
    for k, r in o_grads.items():
        gk = grads[k].double()
        abs_err = float((gk - r).norm())
        err = abs_err / max(float(r.norm()), floor)
        ratio = float(gk.norm()) / max(float(r.norm()), 1e-30)
        if err <= 0.10 and (float(r.norm()) < floor or 0.94 <= ratio <= 1.06):
            continue
        if emu is None:   # the bf16-emulated oracle's own error bounds an ill-conditioned gradient (2.5x allowance)
            emu = {}
            for p in parts:
                _, _, eg = run_oracle(cfg, p, sd=sd, backward=True, bf16_emulation=True)
                for kk, v in eg.items():
                    emu[kk] = emu.get(kk, 0) + v.double() / G
        if abs_err > 2.5 * float((emu[k] - r).norm()):
            bad.append((k, round(err, 4), round(ratio, 4)))
    assert not bad, bad[:12]


# ---------------------------------------------------------------------------------------------------------
# kernels
def _holder():
    class Holder(torch.nn.Module):
        pass
    return Holder()


def _src_params(H, g):
    pos = (0.05 * torch.randn(64, H, device=DEV, generator=g)).requires_grad_()
    typ = (0.05 * torch.randn(2, H, device=DEV, generator=g)).requires_grad_()
    gamma = (1 + 0.1 * torch.randn(H, device=DEV, generator=g)).requires_grad_()
    beta = (0.1 * torch.randn(H, device=DEV, generator=g)).requires_grad_()
    return [pos, typ, gamma, beta]


def _pairs(G, Na, Nb):
    """(text, video) rows of every sequence of the grouped pairing, in sequence order"""
    Gt, Gv = Na // G, Nb // G
    ii, jj = [], []
    for g in range(G):
        for i in range(Gt):
            for j in range(Gv):
                ii.append(g * Gt + i)
                jj.append(g * Gv + j)
    return torch.tensor(ii, device=DEV), torch.tensor(jj, device=DEV)


def _embed(a, b, Na, W, Nb, F, groups, ws, dy, p):
    a = a.detach().clone().requires_grad_()
    b = b.detach().clone().requires_grad_()
    ws = [t.detach().clone().requires_grad_() for t in ws]
    with rt.use_model(_HOLDER, torch.device("cuda", torch.cuda.current_device())) as arena:
        arena.stream_counter = 0
        arena.rng_state[1] = 3
        y = ops.EmbedSrcFn.apply(a, b, Na, W, Nb, F, groups, *ws, p, True)
        y.backward(dy)
    return y.detach(), a.grad, b.grad, [t.grad for t in ws]


_HOLDER = _holder()


@pytest.mark.parametrize("G,Na,Nb", [(1, 3, 4), (2, 4, 6), (3, 6, 6), (4, 8, 4)])
def test_embed_src_grouped_pairs(G, Na, Nb):
    """forward: the bits of aligned mode on explicitly gathered pairs (dropout included).  Backward: each source row's
    gradient is the bits of an all-pairs call on its own micro-batch, and the sum of the expanded form's per-pair
    gradients within bf16 rounding"""
    H, W, F, p = 768, 5, 7, 0.1
    g = torch.Generator(device=DEV).manual_seed(G * 10 + Na)
    a = _bf(torch.randn(Na * W, H, device=DEV, generator=g))
    b = _bf(torch.randn(Nb * F, H, device=DEV, generator=g))
    ws = _src_params(H, g)
    ii, jj = _pairs(G, Na, Nb)
    n_seq = ii.numel()
    dy = _bf(torch.randn(n_seq * (W + F), H, device=DEV, generator=g))
    y, da, db, dws = _embed(a, b, Na, W, Nb, F, G, ws, dy, p)
    a_x = a.view(Na, W, H)[ii].reshape(-1, H)
    b_x = b.view(Nb, F, H)[jj].reshape(-1, H)
    y_x, da_x, db_x, dws_x = _embed(a_x, b_x, n_seq, W, n_seq, F, False, ws, dy, p)
    assert torch.equal(y, y_x)
    if G == 1:   # the plain all-pairs call
        y1, da1, db1, _ = _embed(a, b, Na, W, Nb, F, True, ws, dy, p)
        assert torch.equal(y, y1) and torch.equal(da, da1) and torch.equal(db, db1)
    # the expanded form's per-pair gradients summed over each source row's pairs
    for got, per_pair, idx, n, L in ((da, da_x, ii, Na, W), (db, db_x, jj, Nb, F)):
        ref = torch.zeros(n, L, H, dtype=torch.float64, device=DEV).index_add_(0, idx, per_pair.double().view(-1, L, H))
        mag = torch.zeros_like(ref).index_add_(0, idx, per_pair.double().abs().view(-1, L, H))
        assert ((got.double().view(n, L, H) - ref).abs() <= 2.0 ** -7 * mag + 1e-6).all()
    for t, t_x in zip(dws, dws_x):
        assert (t - t_x).abs().max() <= 1e-4 * max(1.0, float(t_x.abs().max()))
    # each micro-batch alone through the all-pairs kernel: the same source-row gradient bits
    Gt, Gv = Na // G, Nb // G
    T = Gt * Gv * (W + F)
    _, dag, dbg, _ = _embed(a, b, Na, W, Nb, F, G, ws, dy, 0.0)
    for k in range(G):
        _, dak, dbk, _ = _embed(a[k * Gt * W:(k + 1) * Gt * W], b[k * Gv * F:(k + 1) * Gv * F], Gt, W, Gv, F, True, ws,
                                dy[k * T:(k + 1) * T].contiguous(), 0.0)
        assert torch.equal(dag[k * Gt * W:(k + 1) * Gt * W], dak)
        assert torch.equal(dbg[k * Gv * F:(k + 1) * Gv * F], dbk)


def _group_masks(G, Na, Nb, W, F, seed):
    gl = torch.Generator().manual_seed(seed)
    ma = (torch.arange(W).unsqueeze(0) < torch.randint(1, W + 1, (Na, 1), generator=gl)).long().to(DEV)
    mb = (torch.arange(F).unsqueeze(0) < torch.randint(1, F + 1, (Nb, 1), generator=gl)).long().to(DEV)
    ii, jj = _pairs(G, Na, Nb)
    full = torch.cat([ma[ii], mb[jj]], -1).contiguous()
    return ma, mb, full


@pytest.mark.parametrize("G,Na,Nb,W,F", [(2, 4, 6, 16, 12), (3, 6, 3, 48, 64), (2, 4, 4, 100, 200)])
def test_attention_grouped_masks_match_expanded(G, Na, Nb, W, F):
    """attention core (S <= 256) and key-tiled core (S > 256), forward and backward, bit for bit against the expanded
    per-sequence mask"""
    H = 768
    ma, mb, full = _group_masks(G, Na, Nb, W, F, seed=G + W)
    S, n_seq = W + F, full.shape[0]
    g = torch.Generator(device=DEV).manual_seed(5)
    x = _bf(torch.randn(n_seq * S, 3 * H, device=DEV, generator=g))
    q, k, v = x[:, :H], x[:, H:2 * H], x[:, 2 * H:]
    d_o = _bf(torch.randn(n_seq * S, H, device=DEV, generator=g))
    outs = []
    for spec in (ops.MaskSpec(ma, mb, all_pairs=G), ops.MaskSpec(full)):
        o, lse = ops.attention_fwd(q, k, v, n_seq, S, S, spec)
        d = torch.empty_like(x)
        ops.attention_bwd(q, k, v, o, lse, d_o, d[:, :H], d[:, H:2 * H], d[:, 2 * H:], n_seq, S, S, spec)
        outs.append((o, lse, d))
    for a, c in zip(*outs):
        assert torch.equal(a, c)


@pytest.mark.parametrize("G,Na,Nb,W,F", [(2, 4, 6, 16, 16), (3, 6, 6, 48, 64)])
def test_fused_attention_grouped_masks_match_expanded(G, Na, Nb, W, F):
    H = 768
    ma, mb, full = _group_masks(G, Na, Nb, W, F, seed=3 * G + W)
    S, n_seq = W + F, full.shape[0]
    x, w, b, _ = _fused_inputs(n_seq, S, 11)
    d_o = _bf(torch.randn(n_seq * S, H, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3)))
    outs = []
    for spec in (ops.MaskSpec(ma, mb, all_pairs=G), ops.MaskSpec(full)):
        o, lse, qkv = ops.fused_qkv_attention_fwd(x, w, b, n_seq, S, spec)
        dqkv = torch.empty_like(qkv)
        dbias = torch.zeros(3 * H, device=DEV)
        ops.fused_attention_bwd(qkv, o, lse, d_o, dqkv, n_seq, S, spec, dbias=dbias)
        outs.append((o, lse, dqkv, dbias))
    for a, c in zip(*outs):
        assert torch.equal(a, c)


# ---- similarity and losses against fp64 per group ----------------------------------------------------------------
def _maxmargin64(s, margin, n_pair, w_same, w_diff):
    B = s.shape[0]
    d = s.diag()
    w = torch.ones(B, B, dtype=torch.float64, device=s.device)
    if n_pair > 0:
        blk = torch.arange(B, device=s.device) // n_pair
        same = blk.unsqueeze(0) == blk.unsqueeze(1)
        w = torch.where(same, torch.full_like(w, w_same), torch.full_like(w, w_diff))
    return (w * (torch.relu(margin + s - d.view(-1, 1)) + torch.relu(margin + s - d.view(1, -1)))).mean()


def _crossen64(s):
    return -torch.log_softmax(s, -1).diag().mean()


def _milnce64(s, bs, P):
    N = bs * P
    mm_mask = torch.block_diag(*[torch.ones(P, P, dtype=torch.float64, device=s.device)] * bs)
    from_text = torch.cat([s.t(), s - mm_mask * 1e12], 1)   # reference until_module.py:201-221 layout
    pick = torch.arange(bs, device=s.device) * P + P // 2
    rows = from_text[pick]
    pos_mask = torch.cat([mm_mask, torch.zeros_like(mm_mask)], 1)[pick]
    lse = torch.logsumexp(rows, 1)
    lsep = torch.logsumexp(rows.masked_fill(pos_mask == 0, float("-inf")), 1)
    return (lse - lsep).mean()


def _loss_module(kind, bs, n_pair):
    from univl_b200.modules.until_module import CrossEn, MaxMarginRankingLoss, MILNCELoss
    if kind == "maxmargin":
        return MaxMarginRankingLoss(margin=0.1, negative_weighting=1, batch_size=bs, n_pair=n_pair,
                                    hard_negative_rate=0.5)
    if kind == "milnce":
        return MILNCELoss(batch_size=bs, n_pair=n_pair)
    return CrossEn()


@pytest.mark.parametrize("kind", ["maxmargin", "crossen", "milnce"])
@pytest.mark.parametrize("G,bs,n_pair", [(3, 4, 1), (4, 2, 3), (2, 5, 3)])
def test_grouped_sim_losses_fp64(kind, G, bs, n_pair):
    B, H = bs * n_pair, 64
    g = torch.Generator(device=DEV).manual_seed(G * 100 + B)
    t = torch.randn(G * B, H, device=DEV, generator=g).requires_grad_()
    v = torch.randn(G * B, H, device=DEV, generator=g).requires_grad_()
    fn = _loss_module(kind, bs, n_pair)
    sim = ops.SimMatmulFn.apply(t, v, G)
    assert sim.shape == (G, B, B)
    loss = fn(sim)
    loss.backward()
    t64, v64 = t.detach().double(), v.detach().double()
    sim64 = sim.detach().double().requires_grad_()   # the loss reference starts from the kernel's own fp32 sim
    terms = []
    for k in range(G):
        tk, vk = t64[k * B:(k + 1) * B], v64[k * B:(k + 1) * B]
        assert (sim[k].double() - tk @ vk.t()).abs().max() <= 4 * H * U32 * float((tk.abs() @ vk.abs().t()).max())
        s = sim64[k]
        if kind == "maxmargin":
            terms.append(_maxmargin64(s, fn.margin, n_pair if fn.weighted else 0, fn.w_same, fn.w_diff))
        elif kind == "crossen":
            terms.append(_crossen64(s))
        else:
            terms.append(_milnce64(s, bs, n_pair))
    ref = sum(terms) / G
    ref.backward()
    assert abs(float(loss) - float(ref)) <= 1e-5 * max(1.0, float(ref.abs())), (float(loss), float(ref))
    ds = sim64.grad
    dt = torch.cat([ds[k] @ v64[k * B:(k + 1) * B] for k in range(G)])
    dv = torch.cat([ds[k].t() @ t64[k * B:(k + 1) * B] for k in range(G)])
    for got, r in ((t.grad, dt), (v.grad, dv)):
        assert (got.double() - r).abs().max() <= 1e-5 * max(1e-3, float(r.abs().max())), kind
    # G = 1: the [1, B, B] stack gives the bits of today's [B, B] call, loss and gradient
    s1 = sim[:1].detach().clone().requires_grad_()
    s2 = sim[0].detach().clone().requires_grad_()
    l1, l2 = fn(s1), fn(s2)
    l1.backward()
    l2.backward()
    assert torch.equal(l1, l2) and torch.equal(s1.grad[0], s2.grad)
    # one micro-batch's matrix through the grouped loss = its own loss (up to the fp32 mean over groups)
    tg = t.detach()[:B].contiguous()
    vg = v.detach()[:B].contiguous()
    assert torch.equal(ops.SimMatmulFn.apply(tg, vg, 1), sim[0].detach())


def _xent_inputs(G, R, V, K, seed, empty_group=None):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = _bf(torch.randn(G * R, K, device=DEV, generator=g))
    W = (0.05 * torch.randn(V, K, device=DEV, generator=g))
    labels = torch.randint(0, V, (G * R,), device=DEV, generator=g)
    labels[torch.rand(G * R, device=DEV, generator=g) < 0.5] = -1
    labels[::R] = 1
    if empty_group is not None:
        labels[empty_group * R:(empty_group + 1) * R] = -1
    return x, W, labels


def _ref_xent64(logits64, labels, rows):
    out = []
    for r in rows:
        lab = labels[r]
        keep = lab != -1
        if not bool(keep.any()):
            out.append(torch.tensor(float("nan"), dtype=torch.float64, device=DEV))
            continue
        out.append(torch.nn.functional.cross_entropy(logits64[r][keep], lab[keep]))
    return out


def test_grouped_vocab_xent_fp64_and_empty_group():
    G, R, V, K = 3, 40, 1000, 64
    x, W, labels = _xent_inputs(G, R, V, K, seed=1)
    with rt.use_model(_HOLDER, torch.device("cuda", torch.cuda.current_device())):
        xr = x.clone().requires_grad_()
        loss = ops.ProjXentFn.apply(xr, W.to(torch.bfloat16), None, labels, None, 0, False, False, G)
        loss.backward()
    logits = x.double() @ W.to(torch.bfloat16).double().t()
    logits.requires_grad_()
    terms = _ref_xent64(logits, labels, [slice(k * R, (k + 1) * R) for k in range(G)])
    ref = sum(terms) / G
    ref.backward()
    assert abs(float(loss) - float(ref)) <= 1e-5 * max(1.0, float(ref))
    dref = logits.grad @ W.to(torch.bfloat16).double()
    assert (xr.grad.double() - dref).abs().max() <= 2.0 ** -7 * float(dref.abs().max())
    # G = 1 is the ungrouped call; a group without a labelled row makes the loss NaN, as its micro-batch's loss is
    x, W, labels = _xent_inputs(G, R, V, K, seed=2, empty_group=1)
    with rt.use_model(_HOLDER, torch.device("cuda", torch.cuda.current_device())):
        assert torch.isnan(ops.ProjXentFn.apply(x, W.to(torch.bfloat16), None, labels, None, 0, False, False, G))
        assert not torch.isnan(ops.ProjXentFn.apply(x, W.to(torch.bfloat16), None, labels, None, 0, False, False, 1))


def test_grouped_mfm_nce_fp64():
    """target_mode 1: each group's frames are scored against that group's own Tg frames, with the pad mask inside the
    group"""
    G, Tg, K = 3, 48, 1024
    g = torch.Generator(device=DEV).manual_seed(9)
    x = _bf(torch.randn(G * Tg, K, device=DEV, generator=g))
    frames = _bf(0.05 * torch.randn(G * Tg, K, device=DEV, generator=g))
    vm = (torch.rand(G * Tg, device=DEV, generator=g) < 0.8).long()
    labels = torch.where((torch.rand(G * Tg, device=DEV, generator=g) < 0.3) & (vm != 0),
                         torch.arange(G * Tg, device=DEV) % Tg, torch.full((G * Tg,), -1, device=DEV))
    labels[::Tg] = 0
    vm[::Tg] = 1
    with rt.use_model(_HOLDER, torch.device("cuda", torch.cuda.current_device())):
        xr, fr = x.clone().requires_grad_(), frames.clone().requires_grad_()
        loss = ops.ProjXentFn.apply(xr, fr, None, labels, vm, 1, False, False, G)
        loss.backward()
    x64, f64 = x.double().requires_grad_(), frames.double().requires_grad_()
    terms = []
    for k in range(G):
        rows = slice(k * Tg, (k + 1) * Tg)
        m = vm[rows].double()
        lg = x64[rows] @ f64[rows].t() + (1.0 - m.view(-1, 1) * m.view(1, -1)) * -1e8
        sel = labels[rows] != -1
        terms.append(torch.nn.functional.cross_entropy(lg[sel], torch.arange(Tg, device=DEV)[sel]))
    ref = sum(terms) / G
    ref.backward()
    assert abs(float(loss) - float(ref)) <= 1e-4 * max(1.0, float(ref))
    for got, r in ((xr.grad, x64.grad), (fr.grad, f64.grad)):
        assert (got.double() - r).abs().max() <= 2.0 ** -7 * float(r.abs().max())


# ---------------------------------------------------------------------------------------------------------
# determinism
def _step(model, opt, batch, G, reserve=0):
    opt.zero_grad()
    loss = model(**batch, micro_batches=G)
    rt.reserve_sms(reserve)
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


@pytest.mark.parametrize("mode,n_pair", [("ft_align", 1), ("pretrain2", 3)])
def test_grouped_step_deterministic(mode, n_pair):
    G = 3
    cfg = _cfg(mode, n_pair, max_words=24, max_frames=16)
    sd = synth.make_state_dict(cfg, seed=2)
    batch = to_device(_window(cfg, G, seed=5)[0])
    runs = []
    for reserve in (0, 0, 40):
        model, opt = _model_and_opt(cfg, sd, dropout=0.1)
        runs.append([_state(_step(model, opt, batch, G, reserve), opt) for _ in range(2)])
        del model, opt
    assert not torch.equal(runs[0][0]["params"], runs[0][1]["params"])
    for r in (1, 2):
        for s in range(2):
            for k in runs[0][s]:
                assert torch.equal(runs[0][s][k], runs[r][s][k]), (r, s, k)


def test_grouped_step_graph_replay_bitwise():
    G = 3
    cfg = _cfg("ft_align", max_words=24, max_frames=16)
    sd = synth.make_state_dict(cfg, seed=4)
    batch = to_device(_window(cfg, G, seed=6)[0])
    model, opt = _model_and_opt(cfg, sd, dropout=0.1)
    arena = opt.flat.arena
    rng0 = torch.tensor([SEED, 7], dtype=torch.int64, device=DEV)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            _step(model, opt, batch, G)
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
    eager = _state(_step(model, opt, batch, G), opt)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static_loss = _step(model, opt, batch, G)
    restore()
    graph.replay()
    replay = _state(static_loss, opt)
    for k in eager:
        assert torch.equal(eager[k], replay[k]), k


# ---------------------------------------------------------------------------------------------------------
# argument errors
def test_grouped_loss_size_errors():
    from univl_b200.modules.until_module import MaxMarginRankingLoss, MILNCELoss
    sim = torch.zeros(2, 6, 6, device=DEV)
    with pytest.raises(ValueError, match="batch_size"):
        MILNCELoss(batch_size=3, n_pair=3)(sim)
    with pytest.raises(ValueError, match="batch_size"):
        MaxMarginRankingLoss(batch_size=2, n_pair=1)(sim)
    with pytest.raises(ValueError):
        MILNCELoss(batch_size=2, n_pair=3)(torch.zeros(2, 6, 5, device=DEV))
    assert torch.isfinite(MILNCELoss(batch_size=2, n_pair=3)(sim))


def test_micro_batches_argument_errors():
    cfg = _cfg("ft_joint")
    batch = to_device(_window(cfg, 3, seed=1)[0])
    model = build_model(cfg, sd=synth.make_state_dict(cfg, seed=1))
    for bad in (0, -1, 2.0, True):
        with pytest.raises(ValueError, match="micro_batches"):
            model(**batch, micro_batches=bad)
    with pytest.raises(ValueError, match="divide"):
        model(**batch, micro_batches=4)
