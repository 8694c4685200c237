"""Generate tests/golden/*.pt from the UNMODIFIED reference (authoring container only).

TEST INFRASTRUCTURE.  Imports microsoft/UniVL from /root/reference (read-only), loads the deterministic synthetic
weights of oracle/synth.py through the reference's own `init_preweight`, runs `UniVL.forward` + backward in
train mode with every dropout p forced to 0 (SURVEY.md §4 determinism recipe) and stores losses, similarity
matrices, hidden-state slices/checksums and per-parameter gradient norms.  The fixtures are small (no weights:
both sides regenerate them from the seed) and travel to the GPU box, where /root/reference does not exist.

Usage:  python oracle/make_golden.py            (writes tests/golden/ref_<name>.pt for every case below)
"""
import json
import os
import sys
import tempfile
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
from oracle import synth  # noqa: E402

REFERENCE = os.environ.get("UNIVL_REFERENCE", "/root/reference")

# name -> (task_config kwargs, batch kwargs)
CASES = {
    # BASELINE.json configs[0]: retrieval forward+loss, bert-base + 6-layer visual, batch 4, W=F=48
    "cfg1_ft_joint": (dict(mode="ft_joint", batch_size=4), dict(seed=1234, ragged=True)),
    "cfg1_ft_joint_fixedlen": (dict(mode="ft_joint", batch_size=4), dict(seed=1235, ragged=False)),
    "cfg1_ft_align": (dict(mode="ft_align", batch_size=4), dict(seed=1234, ragged=True)),
    # the same two with the reference's own init law (N(0,0.02), zero biases, unit LN): "random-init bert-base"
    "cfg1_ft_joint_init": (dict(mode="ft_joint", batch_size=4), dict(seed=1234, ragged=True), dict(init_law=True)),
    "cfg1_ft_align_init": (dict(mode="ft_align", batch_size=4), dict(seed=1234, ragged=True), dict(init_law=True)),
    "ft_joint_npair2": (dict(mode="ft_joint", batch_size=3, n_pair=2, text_layers=2, visual_layers=1, max_words=16,
                             max_frames=12), dict(seed=7, ragged=True)),
    "caption_small": (dict(mode="caption", batch_size=2, text_layers=2, visual_layers=1, cross_layers=1,
                           decoder_layers=2, max_words=16, max_frames=12), dict(seed=11, ragged=True)),
    "pretrain2_small": (dict(mode="pretrain2", batch_size=3, text_layers=2, visual_layers=1, cross_layers=1,
                             decoder_layers=1, max_words=16, max_frames=12), dict(seed=13, ragged=True)),
    "pretrain1_mil": (dict(mode="pretrain1", batch_size=2, n_pair=3, text_layers=1, visual_layers=1, max_words=16,
                           max_frames=12), dict(seed=17, ragged=True)),
    # ---- BASELINE.json configs[1], [3], [4] at their REAL shapes and full 12/6/2/3 depth (per-rank batch reduced so
    # the CPU reference finishes in minutes; sequence lengths, depths and objectives are the configs' own) ----
    # configs[1]: retrieval fine-tune FT-Align, per-GPU batch 32 (1024 pair sequences), reference init law
    "cfg2_ft_align_b32_init": (dict(mode="ft_align", batch_size=32), dict(seed=1234, ragged=True),
                               dict(init_law=True)),
    # configs[3]: caption stage-two, max_words=128 max_frames=96 (decoder L=128 over S_e=224 encoder tokens)
    "cfg4_caption": (dict(mode="caption", batch_size=2, max_words=128, max_frames=96), dict(seed=21, ragged=True)),
    # configs[4]: pretrain stage-two, all five objectives, W=F=48; n_pair 1 (stress weights) and 3 (init law)
    "cfg5_pretrain2": (dict(mode="pretrain2", batch_size=4), dict(seed=23, ragged=True)),
    "cfg5_pretrain2_npair3_init": (dict(mode="pretrain2", batch_size=4, n_pair=3), dict(seed=29, ragged=True),
                                   dict(init_law=True)),
}

BERT_BASE = dict(attention_probs_dropout_prob=0.1, hidden_act="gelu", hidden_dropout_prob=0.1, hidden_size=768,
                 initializer_range=0.02, intermediate_size=3072, max_position_embeddings=512,
                 num_attention_heads=12, num_hidden_layers=12, type_vocab_size=2, vocab_size=30522)


def import_reference():
    """boto3/botocore are imported at the top of modules/file_utils.py:20-21 and absent here: stub them."""
    for name in ("boto3", "botocore", "botocore.exceptions"):
        if name not in sys.modules:
            sys.modules[name] = types.ModuleType(name)
    sys.modules["botocore.exceptions"].ClientError = type("ClientError", (Exception,), {})
    sys.modules["botocore"].exceptions = sys.modules["botocore.exceptions"]
    if REFERENCE not in sys.path:
        sys.path.insert(0, REFERENCE)
    from modules.modeling import UniVL  # noqa
    return UniVL


def build_reference_model(cfg, state_dict):
    UniVL = import_reference()
    d = tempfile.mkdtemp(prefix="univl_bert_base_")
    with open(os.path.join(d, "bert_config.json"), "w") as fh:
        json.dump(BERT_BASE, fh)
    # reference modules/until_config.py:42 — an absolute path passes through os.path.join unchanged
    model = UniVL.from_pretrained(d, "visual-base", "cross-base", "decoder-base",
                                  state_dict={k: v.clone() for k, v in state_dict.items()}, task_config=cfg)
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    model.train()
    return model


def run_reference(cfg, batch_kwargs, seed=0, weight_kwargs=None):
    sd = synth.make_state_dict(cfg, seed=seed, **(weight_kwargs or {}))
    model = build_reference_model(cfg, sd)
    # every synthetic key must have landed (no silent "missing key" in the non-strict loader)
    msd = model.state_dict()
    for k, v in sd.items():
        assert k in msd and torch.equal(msd[k], v), "key not loaded: " + k
    assert set(msd.keys()) == set(sd.keys()), sorted(set(msd.keys()) ^ set(sd.keys()))[:10]
    batch = synth.make_batch(cfg, **batch_kwargs)
    captured = {}
    hooks = []
    if model.cross is not None and not getattr(cfg, "stage_two", False):
        pass
    orig_sim = model.get_similarity_logits

    def sim_spy(*a, **k):
        out = orig_sim(*a, **k)
        captured.setdefault("sim_matrices", []).append(out.detach().clone())
        return out
    model.get_similarity_logits = sim_spy
    orig_svo = model.get_sequence_visual_output

    def svo_spy(*a, **k):
        s, v = orig_svo(*a, **k)
        captured.setdefault("seq", []).append(s.detach().clone())
        captured.setdefault("vis", []).append(v.detach().clone())
        return s, v
    model.get_sequence_visual_output = svo_spy
    loss = model(**batch)
    loss.backward()
    grads = {}
    seen = set()
    for name, p in model.named_parameters():
        if p.grad is None or id(p) in seen:
            continue
        seen.add(id(p))
        grads[name] = p.grad.detach()
    for h in hooks:
        h.remove()
    return model, sd, batch, float(loss.detach()), captured, grads


def summarise(t):
    t = t.double()
    return dict(sum=float(t.sum()), abs_sum=float(t.abs().sum()), sq_sum=float((t * t).sum()), shape=list(t.shape))


def make_case(name):
    case = CASES[name]
    cfg_kw, batch_kw = case[0], case[1]
    weight_kw = case[2] if len(case) > 2 else {}
    cfg = synth.task_config(**cfg_kw)
    model, sd, batch, loss, cap, grads = run_reference(cfg, batch_kw, weight_kwargs=weight_kw)
    seq, vis = cap["seq"][0], cap["vis"][0]
    gold = dict(
        name=name, cfg_kwargs=cfg_kw, batch_kwargs=batch_kw, weight_seed=0, weight_kwargs=weight_kw, loss=loss,
        torch_version=torch.__version__,
        sim_matrices=[s.float() for s in cap.get("sim_matrices", [])],
        seq_slice=seq[:, :6, :16].clone(), vis_slice=vis[:, :6, :16].clone(),
        seq_summary=summarise(seq), vis_summary=summarise(vis),
        grad_norms={k: float(g.double().norm()) for k, g in grads.items()},
        small_grads={k: g.clone() for k, g in grads.items() if g.numel() <= 1024 and
                     ("layer.0." in k or "embeddings" in k or "similarity" in k or "normalize" in k)},
        n_state_keys=len(model.state_dict()),
    )
    out = os.path.join(ROOT, "tests", "golden", "ref_%s.pt" % name)
    torch.save(gold, out)
    print("%-28s loss %.9f  keys %d  grads %d  -> %s (%.1f KB)" % (name, loss, gold["n_state_keys"], len(grads),
                                                                  out, os.path.getsize(out) / 1024))
    return gold


def _compact(t):
    """full tensor when small; head / tail slices + moments for long ones (keeps the fixture small)"""
    t = t.detach().clone()
    if t.numel() <= 20000:
        return t
    f = t.flatten().double()
    return dict(head=t.flatten()[:256].clone(), tail=t.flatten()[-256:].clone(), sum=float(f.sum()),
                sq_sum=float((f * f).sum()), numel=t.numel())


def make_bert_adam_golden(steps=4):
    """tests/golden/ref_bert_adam.pt: the reference's OWN BertAdam class (modules/optimization.py:66-168) run for
    `steps` steps on a small parameter set arranged in the 4 groups the drivers build (main_task_retrieval.py:173-190:
    decay / no-decay x "bert." / other, lr scaled by coef_lr for "bert." names), preceded each step by the driver's
    clip_grad_norm_(parameters, 1.0) (main_task_retrieval.py:347).  Stores initial values, per-step gradients and the
    parameters + moments after every step, and the reference optimizer's state_dict() after step 3 (so that
    load_state_dict + one more step must reproduce step 4: the resume path of main_pretrain.py:389)."""
    import copy
    import_reference()
    from modules.optimization import BertAdam
    names_shapes, init, grads, no_grad = synth.adam_case(steps)
    params = {n: torch.nn.Parameter(v.clone()) for n, v in init.items()}
    named = list(params.items())
    no_decay = ["bias", "LayerNorm.bias", "LayerNorm.weight"]
    dec = [(n, p) for n, p in named if not any(nd in n for nd in no_decay)]
    nod = [(n, p) for n, p in named if any(nd in n for nd in no_decay)]
    lr, coef, warmup, t_total = synth.ADAM_CASE_HYPER
    groups = [{"params": [p for n, p in dec if "bert." in n], "weight_decay": 0.01, "lr": lr * coef},
              {"params": [p for n, p in dec if "bert." not in n], "weight_decay": 0.01},
              {"params": [p for n, p in nod if "bert." in n], "weight_decay": 0.0, "lr": lr * coef},
              {"params": [p for n, p in nod if "bert." not in n], "weight_decay": 0.0}]
    opt = BertAdam(groups, lr=lr, warmup=warmup, schedule="warmup_linear", t_total=t_total, weight_decay=0.01,
                   max_grad_norm=1.0)
    after = []
    sd3 = None
    for t in range(steps):
        for n, p in params.items():
            p.grad = grads[t][n].clone() if n in grads[t] else None
        torch.nn.utils.clip_grad_norm_(list(params.values()), 1.0)
        opt.step()
        opt.zero_grad()
        after.append({"params": {n: _compact(p.detach()) for n, p in params.items()},
                      "next_m": {n: _compact(opt.state[p]["next_m"]) for n, p in params.items() if p in opt.state},
                      "next_v": {n: _compact(opt.state[p]["next_v"]) for n, p in params.items() if p in opt.state}})
        if t == 2:
            sd3 = copy.deepcopy(opt.state_dict())
            for st in sd3["state"].values():     # the long tensor is regenerated by the test from after[2] ... keep small
                for k in ("next_m", "next_v"):
                    if st[k].numel() > 20000:
                        st[k] = None
    # steps 3-4 go to a continuation file (tests/oracle_util.load_golden) so that no golden file exceeds 1 MB
    gold = dict(names_shapes=names_shapes, after=after[:2], after_parts=["ref_bert_adam_steps3_4.pt"], lr=lr,
                coef_lr=coef, warmup=warmup, t_total=t_total, weight_decay=0.01, max_grad_norm=1.0, global_clip=1.0,
                no_decay=no_decay, state_dict_after3=sd3, torch_version=torch.__version__)
    out = os.path.join(ROOT, "tests", "golden", "ref_bert_adam.pt")
    torch.save(gold, out)
    torch.save({"after": after[2:]}, os.path.join(ROOT, "tests", "golden", "ref_bert_adam_steps3_4.pt"))
    print("bert_adam golden: %d steps -> %s (%.1f KB)" % (steps, out, os.path.getsize(out) / 1024))


if __name__ == "__main__":
    torch.manual_seed(0)
    names = sys.argv[1:] or list(CASES) + ["bert_adam"]
    for n in names:
        if n == "bert_adam":
            make_bert_adam_golden()
        else:
            make_case(n)
