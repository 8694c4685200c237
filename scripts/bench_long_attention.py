"""Time the key-tiled attention core (csrc/attention_long.cu) and the caption workload that needs it.

Prints one JSON line per measurement:
  - forward / backward ms and TFLOP/s of the long kernel on cross-encoder self-attention at S = 288, 512, 1024;
  - the same for the long kernel called directly at S = 256, beside attention.cu at S = 256 (the cost of tiling);
  - `bench.py --mode caption --max_words 128` samples/s at --max_frames 160 (cross S = 288, long kernel) and at 96
    (cross S = 224, attention.cu).
FLOPs are algorithmic: forward 2 products of 2 * Sq * Sk * 64 per (sequence, head) (Q K^T, P V), backward 5 (S
recomputed, dP, dV, dK, dQ); the backward kernels actually compute 7, because the dq and dk/dv kernels each recompute
S and dP.  Times are CUDA events over --iters launches after --warmup.  The card's name and power limit are printed
with the numbers.

usage: python scripts/bench_long_attention.py [--iters 50] [--tokens 16384] [--no-bench]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from univl_b200 import ops  # noqa: E402
from univl_b200 import runtime as rt  # noqa: E402

H, HEADS = 768, 12
SHORT, LONG = "univl_attention", "univl_attention_long"


def card():
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        out["power_limit_and_max_sm_clock"] = q[0] if q else None
    except (OSError, subprocess.SubprocessError):
        out["power_limit_and_max_sm_clock"] = None
    return out


def fwd_call(entry, q, k, v, n_seq, S, spec, p, rng, stream, o, lse):
    """univl_attention_fwd or univl_attention_long_fwd on self-attention (ops.attention_fwd picks by length, and S = 256
    would always go to attention.cu)"""
    rt.call(entry + "_fwd", q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0),
            o.data_ptr(), o.stride(0), lse.data_ptr(), rt.ptr(spec.a), None, spec.Wa, 0, 0, 0, n_seq, HEADS, S, S, 0,
            0.125, p, rng, stream, None)


def bwd_call(entry, q, k, v, o, lse, d_o, dqkv, n_seq, S, spec, p, rng, stream, db):
    dq, dk, dv = dqkv[:, :H], dqkv[:, H:2 * H], dqkv[:, 2 * H:]
    rt.call(entry + "_bwd", q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0),
            o.data_ptr(), o.stride(0), lse.data_ptr(), d_o.data_ptr(), d_o.stride(0), dq.data_ptr(), dq.stride(0),
            dk.data_ptr(), dk.stride(0), dv.data_ptr(), dv.stride(0), rt.ptr(spec.a), None, spec.Wa, 0, 0, 0, n_seq,
            HEADS, S, S, 0, 0.125, p, rng, stream, 0, db[0].data_ptr(), db[1].data_ptr(), db[2].data_ptr(), None)


def time_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def attention_case(S, n_seq, entry, iters, warmup):
    g = torch.Generator(device="cuda").manual_seed(S)
    qkv = (torch.randn(n_seq * S, 3 * H, device="cuda", generator=g)).to(torch.bfloat16)
    q, k, v = qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:]
    lens = torch.randint(S // 2, S + 1, (n_seq,), device="cuda", generator=g)
    spec = ops.MaskSpec((torch.arange(S, device="cuda").unsqueeze(0) < lens.unsqueeze(1)).long())
    rng = torch.tensor([1, 0], dtype=torch.int64, device="cuda")
    o = torch.empty(n_seq * S, H, dtype=torch.bfloat16, device="cuda")
    lse = torch.empty(n_seq * HEADS * S, dtype=torch.float32, device="cuda")
    fwd_call(entry, q, k, v, n_seq, S, spec, 0.1, rng.data_ptr(), 5, o, lse)
    d_o = torch.randn_like(o)
    dqkv = torch.empty_like(qkv)
    db = torch.zeros(3, H, device="cuda")
    fwd = time_ms(lambda: fwd_call(entry, q, k, v, n_seq, S, spec, 0.1, rng.data_ptr(), 5, o, lse), iters, warmup)
    bwd = time_ms(lambda: bwd_call(entry, q, k, v, o, lse, d_o, dqkv, n_seq, S, spec, 0.1, rng.data_ptr(), 5, db),
                  iters, warmup)
    unit = 2.0 * n_seq * HEADS * S * S * 64
    return {"kernel": "attention_long.cu" if entry.endswith("long") else "attention.cu", "S": S, "n_seq": n_seq,
            "fwd_ms": fwd, "fwd_tflops": 2 * unit / (fwd * 1e-3) / 1e12,
            "bwd_ms": bwd, "bwd_tflops": 5 * unit / (bwd * 1e-3) / 1e12, "dropout": 0.1}


def caption_bench(max_frames, steps, warmup):
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(steps), "--warmup",
           str(warmup), "--mode", "caption", "--max_words", "128", "--max_frames", str(max_frames),
           "--no_cpu_baseline", "--no_e2e", "--profile_steps", "0"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1800)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    if r.returncode != 0 or not lines:
        return {"max_frames": max_frames, "error": r.stderr[-2000:]}
    res = json.loads(lines[-1])
    return {"bench": "caption", "max_words": 128, "max_frames": max_frames, "cross_S": 128 + max_frames,
            "samples_per_s": res["value"], "ms_per_step": res["ms_per_step"], "batch": res["config"]["global_batch"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--tokens", type=int, default=16384, help="tokens per call: n_seq = tokens // S")
    ap.add_argument("--bench_steps", type=int, default=10)
    ap.add_argument("--no-bench", dest="no_bench", action="store_true", help="skip the two bench.py caption runs")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_long_attention.py needs a CUDA device")
    print(json.dumps({"card": card()}), flush=True)
    for S, entry in ((256, SHORT), (256, LONG), (288, LONG), (512, LONG), (1024, LONG)):
        print(json.dumps(attention_case(S, max(1, a.tokens // S), entry, a.iters, a.warmup)), flush=True)
    if not a.no_bench:
        for mf in (96, 160):
            print(json.dumps(caption_bench(mf, a.bench_steps, 3)), flush=True)


if __name__ == "__main__":
    main()
