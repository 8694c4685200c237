"""Does FP8 retrieval evaluation (UNIVL_EVAL_PRECISION=fp8) keep the ranking of a trained cross encoder?

Random-init logits are nearly flat and say little about ranking, so this trains a reduced FT-Align model (2 text
layers, 1 visual layer, 2 cross layers, max-margin loss over in-batch negatives, as main_task_retrieval.py with
--train_sim_after_cross) with this package on a synthetic matched-pair task, then scores held-out pairs under bf16 and
FP8 evaluation.

Task: a text is [CLS] + W - 2 tokens drawn from a vocabulary of --vocab ids + [SEP]; its video's frame f is a fixed
random 1024-d code of the text's token f + 1 plus Gaussian noise (--noise).  Matching a text to its video needs the
cross encoder to compare token content with frame content position by position.

Training runs until bf16 R@1 on the --eval held-out pairs reaches --target-r1 (checked every --eval-every steps) or
--max-steps.  Then both precisions score the held-out text x video matrix, and the script reports R@1/5/10 and median
rank (text -> video, the metric of the reference's compute_metrics), the fraction of texts whose top-1 video changes,
and max |logit difference| / the row's bf16 logit standard deviation.  Prints one JSON line per evaluation and a
final JSON line.

usage: python scripts/eval_fp8_quality.py [--eval 1024] [--batch 64] [--max-steps 4000] [--target-r1 50]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

W, F, VIDEO_DIM = 16, 12, 1024


def make_task(vocab, noise, seed):
    g = torch.Generator().manual_seed(seed)
    codes = torch.randn(vocab, VIDEO_DIM, generator=g)  # the fixed token -> frame map

    def sample(n, seed):
        gs = torch.Generator().manual_seed(seed)
        tok = torch.randint(0, vocab, (n, W - 2), generator=gs)
        ids = torch.empty(n, W, dtype=torch.long)
        ids[:, 0] = 101
        ids[:, 1:W - 1] = tok + 1000
        ids[:, W - 1] = 102
        video = codes[tok[:, :F]] + noise * torch.randn(n, F, VIDEO_DIM, generator=gs)
        ones = torch.ones(n, 1, W, dtype=torch.long)
        return dict(input_ids=ids.view(n, 1, W).cuda(), token_type_ids=torch.zeros_like(ones).cuda(),
                    attention_mask=ones.cuda(), video=video.view(n, 1, F, VIDEO_DIM).cuda(),
                    video_mask=torch.ones(n, 1, F, dtype=torch.long).cuda())

    return sample


def logits(model, data, precision):
    os.environ["UNIVL_EVAL_PRECISION"] = precision
    model.eval()
    with torch.no_grad():
        seq, vis = model.get_sequence_visual_output(data["input_ids"], data["token_type_ids"], data["attention_mask"],
                                                    data["video"], data["video_mask"])
        out = model.get_similarity_logits(seq, vis, data["attention_mask"], data["video_mask"])
    torch.cuda.synchronize()
    return out.float()


def metrics(sim):
    """text -> video: rank of the matching video (1 = best; ties count in its favour)"""
    diag = sim.diagonal().unsqueeze(1)
    rank = (sim > diag).sum(1) + 1
    r = rank.float()
    out = {"R@%d" % k: round(100 * float((r <= k).float().mean()), 2) for k in (1, 5, 10)}
    out["MedR"] = float(r.median())
    return out


def train(a, mode, sample, held_out, evaluate):
    """Train a reduced model of `mode` (2 text layers, 1 visual layer, 2 cross layers, no dropout) with AdamW on the
    task until evaluate(model, held_out)["R@1"] reaches a.target_r1 (checked every a.eval_every steps) or a.max_steps.
    Prints one JSON line per evaluation.  -> (model, steps)"""
    from oracle import synth
    from tests.model_util import build_model

    cfg = synth.task_config(mode=mode, batch_size=a.batch, text_layers=2, visual_layers=1, cross_layers=2,
                            max_words=W, max_frames=F)
    model = build_model(cfg, sd=synth.make_state_dict(cfg, seed=a.seed, init_law=True), dropout=0.0)
    opt = torch.optim.AdamW(model.parameters(), lr=a.lr, weight_decay=0.01)
    warmup = 100
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda s: min(1.0, (s + 1) / warmup))
    step, t0 = 0, time.perf_counter()
    while True:
        model.train()
        loss = model(**sample(a.batch, seed=step))
        opt.zero_grad(set_to_none=True)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(model.parameters(), 1.0)
        opt.step()
        sched.step()
        step += 1
        if step % a.eval_every == 0 or step == a.max_steps:
            m = evaluate(model, held_out)
            print(json.dumps({"mode": mode, "step": step, "loss": round(float(loss.detach()), 4), "bf16": m,
                              "train_s": round(time.perf_counter() - t0, 1)}), flush=True)
            if m["R@1"] >= a.target_r1 or step >= a.max_steps:
                return model, step


def arguments(ap):
    """the task and training options"""
    ap.add_argument("--eval", type=int, default=1024, help="held-out pairs")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--vocab", type=int, default=256)
    ap.add_argument("--noise", type=float, default=0.5)
    ap.add_argument("--lr", type=float, default=1e-4)
    ap.add_argument("--max-steps", type=int, default=4000)
    ap.add_argument("--eval-every", type=int, default=250)
    ap.add_argument("--target-r1", type=float, default=50.0)
    ap.add_argument("--seed", type=int, default=0)
    return ap


def main():
    a = arguments(argparse.ArgumentParser()).parse_args()
    if not torch.cuda.is_available():
        sys.exit("eval_fp8_quality: needs a CUDA device")

    torch.manual_seed(a.seed)
    sample = make_task(a.vocab, a.noise, a.seed + 1)
    held_out = sample(a.eval, seed=10 ** 6)
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "task": vars(a), "W": W, "F": F,
                      "chance_R@1": round(100.0 / a.eval, 3)}), flush=True)
    model, step = train(a, "ft_align", sample, held_out, lambda m, d: metrics(logits(m, d, "bf16")))

    bf16 = logits(model, held_out, "bf16")
    fp8 = logits(model, held_out, "fp8")
    os.environ.pop("UNIVL_EVAL_PRECISION", None)
    d = (fp8 - bf16).abs()
    row_std = bf16.std(dim=1, keepdim=True)
    out = {"steps": step, "batch": a.batch, "held_out_pairs": a.eval, "bf16": metrics(bf16), "fp8": metrics(fp8),
           "top1_changed_fraction": float((fp8.argmax(1) != bf16.argmax(1)).float().mean()),
           "max_abs_dlogit": float(d.max()), "max_abs_dlogit_over_row_std": float((d / row_std).max()),
           "mean_row_std": float(row_std.mean())}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
