"""Time one gradient-accumulation window of UniVL pretraining two ways, at the README's per-GPU pretraining shapes:

  (a) loop:    the reference driver's loop on this package, G x (forward, loss / G, backward, float(loss)), then one
               fused BertAdam step (main_pretrain.py:326-345);
  (b) grouped: one forward(micro_batches=G), one backward, float(loss), the same BertAdam step.

Both compute the same objective: (1/G) sum_g L_g, every micro-batch with its own similarity matrix, negatives and means.
Stage I: b = 15 clips x n_pair 3 = 45 rows per micro-batch, G = 16, text 12 / visual 6 layers (MIL-NCE on mean-pooled
similarity).  Stage II: b = 2 x 3 = 6 rows, G = 60, text 12 / visual 6 / cross 2 / decoder 3 layers, all five objectives.
Words 48, frames 64, dropout 0 (so (a) and (b) see the same network and their losses can be compared).

Per stage: ms per optimizer step and samples/s (G * b * n_pair per step) for (a) and (b), three runs each, alternated in
the same process; the torch allocator's peak memory of each (kernel scratch from the CUDA stream-ordered pool is not
counted); and, before any step, the loss and flat-gradient difference between (a) and (b) on the same parameters.  The
card's name, power limit and SM clock are read in the same call.  Prints one JSON line per stage, then a table.

usage: python scripts/bench_micro_batches.py [--stages 1,2] [--steps 3] [--runs 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

STAGES = {1: dict(mode="pretrain1", b=15, G=16), 2: dict(mode="pretrain2", b=2, G=60)}
N_PAIR, WORDS, FRAMES = 3, 48, 64


def nvsmi(query):
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=" + query, "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else None
    except (OSError, subprocess.SubprocessError):
        return None


def build(stage):
    from oracle import synth
    from tests.model_util import bert_dir
    from univl_b200.modules.modeling import UniVL
    from univl_b200.optim import FusedBertAdam
    s = STAGES[stage]
    # the driver divides batch_size by the accumulation steps before building the model: the losses are built for b
    cfg = synth.task_config(mode=s["mode"], batch_size=s["b"], n_pair=N_PAIR, max_words=WORDS, max_frames=FRAMES)
    torch.manual_seed(0)
    model = UniVL.from_pretrained(bert_dir(), "visual-base", "cross-base", "decoder-base", task_config=cfg)
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    model.to("cuda").train()
    named = list(model.named_parameters())
    no_decay = ["bias", "LayerNorm.bias", "LayerNorm.weight"]
    groups = [{"params": [p for n, p in named if not any(nd in n for nd in no_decay)], "weight_decay": 0.01},
              {"params": [p for n, p in named if any(nd in n for nd in no_decay)], "weight_decay": 0.0}]
    opt = FusedBertAdam(groups, lr=1e-4, warmup=0.1, t_total=100000, max_grad_norm=1.0, model=model)
    opt._build()
    parts = [{k: v.cuda() for k, v in synth.make_batch(cfg, seed=1000 + g).items()} for g in range(s["G"])]
    window = {k: torch.cat([p[k] for p in parts], 0) for k in parts[0]}
    return cfg, model, opt, parts, window


def loop_grads(model, opt, parts):
    opt.zero_grad()
    total = 0.0
    for p in parts:
        loss = model(**p) / len(parts)
        loss.backward()
        total += float(loss)              # the reference loop's per-micro-step host read (main_pretrain.py:338)
    return total


def grouped_grads(model, opt, window, G):
    opt.zero_grad()
    loss = model(**window, micro_batches=G)
    loss.backward()
    return float(loss)


def timed(fn, opt, steps):
    """ms per optimizer step over `steps` steps (device events; the last event is synchronised)"""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        fn()
        opt.step()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / steps


def run_stage(stage, steps, runs):
    s = STAGES[stage]
    G, rows = s["G"], s["b"] * N_PAIR
    cfg, model, opt, parts, window = build(stage)
    arms = {"loop": lambda: loop_grads(model, opt, parts), "grouped": lambda: grouped_grads(model, opt, window, G)}

    # the two arms on the same parameters, before any step
    la = arms["loop"]()
    ga = opt.g.clone()
    lb = arms["grouped"]()
    gb = opt.g.clone()
    torch.cuda.synchronize()
    grad_rel = float((ga - gb).double().norm() / ga.double().norm())

    peak = {}
    for name, fn in arms.items():          # warm-up (and allocator peak) of each arm
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        for _ in range(2):
            fn()
            opt.step()
        torch.cuda.synchronize()
        peak[name] = torch.cuda.max_memory_allocated() / 2 ** 30
    ms = {"loop": [], "grouped": []}
    clocks = []
    for _ in range(runs):
        for name, fn in arms.items():
            ms[name].append(timed(fn, opt, steps))
            clocks.append(nvsmi("clocks.sm"))
    res = {"stage": stage, "mode": s["mode"], "b": s["b"], "n_pair": N_PAIR, "G": G, "rows_per_micro_batch": rows,
           "samples_per_step": G * rows, "layers": [cfg.text_num_hidden_layers, cfg.visual_num_hidden_layers] +
           ([cfg.cross_num_hidden_layers, cfg.decoder_num_hidden_layers] if stage == 2 else []),
           "loss_loop": la, "loss_grouped": lb, "loss_abs_diff": abs(la - lb), "flat_grad_rel_diff": grad_rel,
           "peak_gib": peak, "sm_clock_during": clocks}
    for name in ms:
        res[name + "_ms"] = [round(t, 2) for t in ms[name]]
        res[name + "_samples_per_s"] = [round(G * rows / (t / 1e3), 1) for t in ms[name]]
    res["speedup_median"] = round(sorted(ms["loop"])[len(ms["loop"]) // 2] /
                                  sorted(ms["grouped"])[len(ms["grouped"]) // 2], 2)
    del model, opt, parts, window
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--stages", default="1,2")
    ap.add_argument("--steps", type=int, default=3, help="optimizer steps per timed run")
    ap.add_argument("--runs", type=int, default=3, help="timed runs per arm, alternated")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_micro_batches.py: no CUDA device (the kernels are sm_90a only)")
    card = {"card": torch.cuda.get_device_name(0), "power_limit": nvsmi("power.limit"),
            "sm_clock": nvsmi("clocks.sm"), "max_sm_clock": nvsmi("clocks.max.sm")}
    print(json.dumps(card), flush=True)
    results = []
    for st in [int(x) for x in a.stages.split(",") if x]:
        t0 = time.time()
        r = run_stage(st, a.steps, a.runs)
        r["wall_s"] = round(time.time() - t0, 1)
        results.append(r)
        print(json.dumps(r), flush=True)
    print("| stage | G x rows | way | ms / step (3 runs) | samples/s (median) | peak GiB |")
    print("|---|---|---|---|---|---|")
    for r in results:
        for name in ("loop", "grouped"):
            sps = sorted(r[name + "_samples_per_s"])[len(r[name + "_samples_per_s"]) // 2]
            print("| %s | %d x %d | %s | %s | %.1f | %.1f |" % (
                "I" if r["stage"] == 1 else "II", r["G"], r["rows_per_micro_batch"], name,
                " / ".join("%.1f" % t for t in r[name + "_ms"]), sps, r["peak_gib"][name]))


if __name__ == "__main__":
    main()
