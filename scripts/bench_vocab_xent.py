"""Time and size the vocabulary cross-entropy in both UNIVL_VOCAB_LOSS modes ("logits": fp32 logits kept for backward;
"fused": univl_vocab_xent_fwd / _bwd, no logits in memory).

  head   ProjXentFn forward + backward of the tied 30522-word projection (K = 768, bias, about 30 % of the rows
         unscored) at T = 4096 (the caption step's rows) and T = 17280 (one stage-II pretraining window's MLM or caption
         rows): ms per call from CUDA events, the modes alternated --runs times, and the torch allocator's peak over one
         call above what was allocated before it.
  model  the torch allocator's peak, absolute and above what was allocated before the step, of one caption training
         step (batch 32, 128 words, 96 frames, full depth) and of one stage-II pretraining window (micro_batches =
         60 of 2 x n_pair 3 rows, 48 words, 64 frames), per mode.
  bench  `bench.py --gpus 1 --mode caption --max_words 128 --max_frames 96` and `bench.py --gpus 1 --mode pretrain2`,
         each mode in turn, --runs times (bench.py reads UNIVL_VOCAB_LOSS from its environment).

The card's name, power limit and SM clock are read in the same call.  Prints one JSON line per measurement and writes
them to --out if given.

usage: python scripts/bench_vocab_xent.py [--parts head,model,bench] [--runs 3] [--steps 20]
                                         [--bench_cases caption,pretrain2] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

MODES = ("logits", "fused")
V, K = 30522, 768


def nvsmi(query):
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=" + query, "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else None
    except (OSError, subprocess.SubprocessError):
        return None


def emit(rec, out):
    print(json.dumps(rec), flush=True)
    if out:
        with open(out, "a") as fh:
            fh.write(json.dumps(rec) + "\n")


def head(runs, iters, out):
    from univl_b200 import ops
    from univl_b200 import runtime as rt

    class Head(torch.nn.Module):
        def __init__(self):
            super().__init__()
            g = torch.Generator(device="cuda").manual_seed(0)
            self.weight = torch.nn.Parameter(0.05 * torch.randn(V, K, device="cuda", generator=g))
            self.bias = torch.nn.Parameter(torch.randn(V, device="cuda", generator=g))

    h = Head()
    dev = torch.device("cuda", torch.cuda.current_device())
    for T in (4096, 17280):
        g = torch.Generator(device="cuda").manual_seed(T)
        x = torch.randn(T, K, device="cuda", generator=g).to(torch.bfloat16).requires_grad_()
        labels = torch.randint(0, V, (T,), device="cuda", generator=g)
        labels[torch.rand(T, device="cuda", generator=g) < 0.3] = -1

        def call():
            loss = ops.ProjXentFn.apply(x, h.weight, h.bias, labels, None, 0, True, False, 1)
            loss.backward()
            h.weight.grad = h.bias.grad = x.grad = None

        res = {m: {"ms": []} for m in MODES}
        with rt.use_model(h, dev):
            for m in MODES:  # warm-up and peak memory
                os.environ["UNIVL_VOCAB_LOSS"] = m
                call()
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                call()
                torch.cuda.synchronize()
                res[m]["peak_gib"] = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
            for _ in range(runs):
                for m in MODES:
                    os.environ["UNIVL_VOCAB_LOSS"] = m
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(iters):
                        call()
                    e1.record()
                    torch.cuda.synchronize()
                    res[m]["ms"].append(e0.elapsed_time(e1) / iters)
        os.environ.pop("UNIVL_VOCAB_LOSS", None)
        emit({"part": "head", "T": T, "V": V, "K": K, "runs": res, "sm_clock_mhz": nvsmi("clocks.sm")}, out)


def model(out):
    from oracle import synth
    from tests.model_util import build_model

    cases = [("caption step", synth.task_config(mode="caption", batch_size=32, max_words=128, max_frames=96), 1),
             ("stage-II window", synth.task_config(mode="pretrain2", batch_size=2, n_pair=3, max_words=48,
                                                   max_frames=64), 60)]
    for name, cfg, G in cases:
        parts = [synth.make_batch(cfg, seed=1000 + g) for g in range(G)]
        batch = {k: torch.cat([p[k] for p in parts], 0).cuda() for k in parts[0]}
        kw = {} if G == 1 else {"micro_batches": G}
        rec = {"part": "model", "case": name}
        for m in MODES:
            os.environ["UNIVL_VOCAB_LOSS"] = m
            torch.manual_seed(0)
            net = build_model(cfg, dropout=0.0)
            net(**batch, **kw).backward()  # warm-up
            torch.cuda.synchronize()
            for p in net.parameters():
                p.grad = None
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            loss = net(**batch, **kw)
            loss.backward()
            torch.cuda.synchronize()
            rec[m] = {"step_peak_gib": (torch.cuda.max_memory_allocated() - base) / 2 ** 30,
                      "peak_gib": torch.cuda.max_memory_allocated() / 2 ** 30, "loss": float(loss.detach())}
            del net, loss
            torch.cuda.empty_cache()
        os.environ.pop("UNIVL_VOCAB_LOSS", None)
        emit(rec, out)


def bench(runs, steps, cases, out):
    cmds = {"caption": ["--mode", "caption", "--max_words", "128", "--max_frames", "96"],
            "pretrain2": ["--mode", "pretrain2"]}
    for name in cases:
        extra = cmds[name]
        res = {m: [] for m in MODES}
        for _ in range(runs):
            for m in MODES:
                env = dict(os.environ, UNIVL_VOCAB_LOSS=m)
                cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(steps),
                       "--warmup", "3", "--no_cpu_baseline", *extra]
                p = subprocess.run(cmd, env=env, capture_output=True, text=True, cwd=ROOT)
                lines = [ln for ln in p.stdout.splitlines() if ln.startswith("{")]
                if p.returncode != 0 or not lines:
                    raise RuntimeError("bench.py failed (%d): %s" % (p.returncode, p.stderr[-2000:]))
                rec = json.loads(lines[-1])
                res[m].append(rec["ms_per_step"])
        emit({"part": "bench", "case": name, "ms_per_step": res, "sm_clock_mhz": nvsmi("clocks.sm")}, out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", default="head,model,bench")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20, help="head calls per timed run")
    ap.add_argument("--steps", type=int, default=20, help="bench.py --steps")
    ap.add_argument("--bench_cases", default="caption,pretrain2")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vocab_xent.py measures on a CUDA device; none is available")
    emit({"gpu": nvsmi("name"), "power_limit": nvsmi("power.limit"), "max_sm_clock": nvsmi("clocks.max.sm")}, a.out)
    parts = a.parts.split(",")
    if "head" in parts:
        head(a.runs, a.iters, a.out)
    if "model" in parts:
        model(a.out)
    if "bench" in parts:
        bench(a.runs, a.steps, a.bench_cases.split(","), a.out)


if __name__ == "__main__":
    main()
