"""Where the device time of one FT-Align training step goes, per kernel.

Builds the step bench.py times (FT-Align, 12L text / 6L visual / 2L cross, per-GPU batch 32, 48 words, 48 frames,
dropout 0.1, fused BertAdam), runs it eagerly on one stream (UNIVL_TWO_STREAM=0, as bench.py does for its per-launch
GEMM timings, so kernel durations are not shared with a concurrent stream), and records --steps steps under
torch.profiler with CUDA activities.  Prints, as JSON lines: the card's name, power limit and maximum SM clock; then
per kernel name its device time per step, launches per step and share of the step's kernel time, largest first; then
the total.  The wgmma GEMM's template arguments are <BLOCK_N, STAGES, A MN-major, B MN-major>: the weight gradients
are the instances with both operands MN-major.

usage: python scripts/profile_step.py [--steps 3] [--warmup 3] [--top 40]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ["UNIVL_TWO_STREAM"] = "0"

import torch  # noqa: E402


def nvsmi(query):
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=" + query, "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else None
    except (OSError, subprocess.SubprocessError):
        return None


def build_step(batch):
    """the model, optimizer and seeded device batch of bench.py's default workload; returns step()"""
    from oracle import synth
    from tests.model_util import bert_dir
    from univl_b200.modules.modeling import UniVL
    from univl_b200.optim import FusedBertAdam

    dev = torch.device("cuda", 0)
    cfg = synth.task_config(mode="ft_align", batch_size=batch, n_gpu=1, max_words=48, max_frames=48)
    torch.manual_seed(0)
    model = UniVL.from_pretrained(bert_dir(), "visual-base", "cross-base", "decoder-base", task_config=cfg)
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.1
    model.to(dev).train()
    named = list(model.named_parameters())
    no_decay = ["bias", "LayerNorm.bias", "LayerNorm.weight"]
    dec = [p for n, p in named if not any(nd in n for nd in no_decay)]
    nod = [p for n, p in named if any(nd in n for nd in no_decay)]
    opt = FusedBertAdam([{"params": dec, "weight_decay": 0.01}, {"params": nod, "weight_decay": 0.0}], lr=3e-5,
                        warmup=0.1, t_total=100000, max_grad_norm=1.0, global_clip_norm=1.0, model=model)
    data = {k: v.to(dev) for k, v in synth.make_batch(cfg, seed=1234, b=batch).items()}

    def step():
        opt.zero_grad()
        loss = model(**data)
        loss.backward()
        opt.step()
        return loss
    return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--top", type=int, default=40, help="kernel names printed (the total counts all)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("profile_step.py needs a CUDA device")
    torch.cuda.set_device(0)
    print(json.dumps({"card": torch.cuda.get_device_name(0),
                      "power_limit_and_max_sm_clock": nvsmi("power.limit,clocks.max.sm")}), flush=True)
    step = build_step(a.batch)
    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.steps):
            step()
        torch.cuda.synchronize()
    per = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        t = per.setdefault(ev.name, [0.0, 0])
        t[0] += ev.time_range.elapsed_us()
        t[1] += 1
    total = sum(t for t, _ in per.values())
    for name, (us, n) in sorted(per.items(), key=lambda kv: -kv[1][0])[:a.top]:
        print(json.dumps({"kernel": name[:160], "ms_per_step": round(us / a.steps * 1e-3, 4),
                          "launches_per_step": n / a.steps, "share": round(us / total, 4)}), flush=True)
    print(json.dumps({"total_kernel_ms_per_step": round(total / a.steps * 1e-3, 3),
                      "launches_per_step": sum(n for _, n in per.values()) / a.steps,
                      "sm_clock_after": nvsmi("clocks.sm")}), flush=True)


if __name__ == "__main__":
    main()
