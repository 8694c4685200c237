"""Time one beam step's vocabulary selection at the MSRVTT caption batch (64 instances x 5 beams, R = 320 rows, V = 30522,
K = 768) in two ways, alternated, with CUDA events over many launches:

  fused   univl_vocab_beam_topk: lse pass + selection pass over the vocabulary, no logits in memory, then the merge
  eager   what beam_search runs: the fp32 logits GEMM (cls.logits), torch.log_softmax, + scores, topk over n_beam x V

Both start from the head transform's output x.  Prints one JSON line with the card's name and power limit.

    python scripts/bench_beam_topk.py --iters 200
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


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-inst", type=int, default=64)
    ap.add_argument("--n-beam", type=int, default=5)
    ap.add_argument("--vocab", type=int, default=30522)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: nothing to time")
    dev = "cuda"
    n, nb, V, K = a.n_inst, a.n_beam, a.vocab, 768
    R = n * nb
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(R, K, device=dev, generator=g).to(torch.bfloat16)
    w16 = (0.05 * torch.randn(V, K, device=dev, generator=g)).to(torch.bfloat16)
    bias = torch.randn(V, device=dev, generator=g)
    score = -torch.rand(R, device=dev, generator=g)
    live = torch.full((n,), nb, dtype=torch.int32, device=dev)
    ws = ops.vocab_beam_topk_workspace(n, nb, V, x)
    out = (torch.empty(R, device=dev), torch.empty(n, nb, device=dev),
           torch.empty(n, nb, dtype=torch.int32, device=dev))
    logits = torch.empty((R, ops._ld_pad(V)), dtype=torch.float32, device=dev)[:, :V]

    def fused():
        ops.vocab_beam_topk(x, w16, bias, score, live, nb, ws, out=out)

    def eager():
        ops.gemm(x, w16, R, V, K, logits, epi=ops.EPI_F32, bias=bias)
        lk = (torch.log_softmax(logits, dim=1) + score[:, None]).view(n, nb * V)
        lk.topk(nb, dim=1, largest=True, sorted=True)

    runs = {"fused": fused, "eager": eager}
    for f in runs.values():
        for _ in range(10):
            f()
    times = {k: [] for k in runs}
    for _ in range(a.rounds):
        for name, f in runs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.iters):
                f()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(round(e0.elapsed_time(e1) * 1e3 / a.iters, 1))
    # the GEMM's work, done twice by the fused kernel (lse pass and selection pass)
    flop = 2.0 * R * V * K
    res = {"card": card(), "R": R, "V": V, "K": K, "n_beam": nb, "iters": a.iters,
           "us_per_step": times, "gemm_tflops_once": round(flop / 1e12, 4)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
