"""Time FT-Align retrieval scoring in evaluation (model.eval() under torch.no_grad(), as the reference's eval_epoch runs
get_similarity_logits) at W = F = 48 words / frames and two cross layers, from random bf16 encoder outputs:

  (a) all-pairs: every text x video pair sequence through the cross encoder in one batch
      (UniVL._cross_similarity_all_pairs, the path training uses), at the largest size it holds (--old, default 128);
  (b) tiled:     UniVL._cross_similarity_eval, tiles of at most modeling.EVAL_PAIR_TOKENS pair tokens with the first
                 cross layer's Q/K/V projections computed once per text row and once per video row.

(a) and (b) run alternated in one process at the --old size, then (b) alone at the --sizes, once per evaluation
precision of --precision (UNIVL_EVAL_PRECISION: bf16, or fp8 for the cross layers' dense GEMMs over the pair tokens),
the precisions alternated within every run, after one untimed call of each precision on the first 512 rows.
Per row: ms per call,
pairs/s, achieved TFLOP/s from the algorithmic FLOP counts below, the torch allocator's peak over the call (kernel
scratch from the stream-ordered pool is not counted; the eval path draws none) and, for (b), the part of that peak that
one tile accounts for (peak - the per-source rows - the result), and for a precision other than bf16 the max |logit
difference| against the bf16 result of the same run.  The FLOP count is the algorithmic one for every precision.  Then
one call per size and precision under torch.profiler, in runs of their own, splits the GPU time into GEMM kernels
(gemm_wgmma_kernel, gemm_fp8_kernel) and all other work.  The card's name, power limit and SM clock are read in the
same call.  Prints one JSON line per row, then a table.

FLOPs (multiply-add = 2) per pair at S = W + F, H = 768, I = 3072, L cross layers, the last one token-0 only:
  (L-1) S (8H^2 + 4HI + 4SH)  +  S 4H^2 (last layer K/V)  +  2H^2 + 4SH + 2H^2 + 4HI (last layer, token 0)  +  2H^2
  (pooler); (b) does S 6H^2 less per pair (first layer Q/K/V) and (Nt W + Nv F) 6H^2 once per call.

usage: python scripts/bench_retrieval_eval.py [--old 128] [--sizes 1024,3500] [--runs 3] [--precision bf16,fp8]
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

H, I, W, F, LAYERS = 768, 3072, 48, 48, 2


def nvsmi(query):
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=" + query, "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else None
    except (OSError, subprocess.SubprocessError):
        return None


def flops(Nt, Nv, tiled):
    S = W + F
    per_pair = ((LAYERS - 1) * S * (8 * H * H + 4 * H * I + 4 * S * H) + S * 4 * H * H
                + 2 * H * H + 4 * S * H + 2 * H * H + 4 * H * I + 2 * H * H)
    if not tiled:
        return Nt * Nv * per_pair
    return Nt * Nv * (per_pair - S * 6 * H * H) + (Nt * W + Nv * F) * 6 * H * H


def build():
    from oracle import synth
    from tests.model_util import build_model
    cfg = synth.task_config(mode="ft_align", batch_size=2, text_layers=1, visual_layers=1, cross_layers=LAYERS,
                            max_words=W, max_frames=F)
    return build_model(cfg, seed=0).eval()


def inputs(N, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, W if seed % 2 == 0 else F, H, generator=g).to(torch.bfloat16).cuda()
    L = x.shape[1]
    lens = torch.randint(L // 4, L + 1, (N,), generator=g)
    return x, (torch.arange(L).view(1, L) < lens.view(N, 1)).long().cuda()


def run(model, N, tiled, seq, vis, am, vm, precision="bf16"):
    from univl_b200 import runtime as rt
    os.environ["UNIVL_EVAL_PRECISION"] = precision
    s2, v2 = seq.reshape(-1, H), vis.reshape(-1, H)
    with torch.no_grad(), rt.use_model(model, seq.device):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        if tiled:
            out = model._cross_similarity_eval(s2, v2, am, vm)
        else:
            out = model._cross_similarity_all_pairs(s2, v2, am, vm)
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        peak = torch.cuda.max_memory_allocated() - base
    return out, ms, peak


def profile(model, N, seq, vis, am, vm, precision):
    """GPU time of one tiled call, split into GEMM kernels and everything else"""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity
    with torch.profiler.profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(model, N, True, seq, vis, am, vm, precision)
    gemm = other = 0.0
    for e in prof.key_averages():
        if e.device_type != DeviceType.CUDA:
            continue
        if "gemm" in e.key:
            gemm += e.self_device_time_total
        else:
            other += e.self_device_time_total
    r = dict(profile="tiled", precision=precision, Nt=N, Nv=N, gemm_ms=round(gemm / 1e3, 1),
             other_ms=round(other / 1e3, 1), gemm_share=round(gemm / max(gemm + other, 1e-9), 3))
    print(json.dumps(r), flush=True)
    return r


def row(name, N, tiled, ms, peak, precision="bf16", dlogit=None):
    from univl_b200.modules import modeling
    f = flops(N, N, tiled)
    r = dict(path=name, precision=precision, Nt=N, Nv=N, W=W, F=F, cross_layers=LAYERS, ms=round(ms, 2),
             pairs_per_s=round(N * N / ms * 1e3), tflop=round(f / 1e12, 2), tflop_per_s=round(f / ms / 1e9, 1),
             peak_gib=round(peak / 2 ** 30, 3))
    if tiled:
        per_source = 2 * N * W * (H + 3 * H) * 2   # source embedding rows and their Q/K/V projections
        r["tile_peak_gib"] = round((peak - per_source - N * N * 4) / 2 ** 30, 3)
        r["eval_pair_tokens"] = modeling.EVAL_PAIR_TOKENS
    if dlogit is not None:
        r["max_abs_dlogit_vs_bf16"] = dlogit
    r["sm_clock"] = nvsmi("clocks.sm")
    print(json.dumps(r), flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--old", type=int, default=128)
    ap.add_argument("--sizes", default="1024,3500")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--precision", default="bf16", help="comma-separated eval precisions of the tiled path: bf16,fp8")
    a = ap.parse_args()
    precisions = [p for p in a.precision.split(",") if p]
    if "bf16" not in precisions:
        precisions.insert(0, "bf16")  # the reference result of the logit differences
    if not torch.cuda.is_available():
        sys.exit("bench_retrieval_eval: needs a CUDA device")
    print(json.dumps({"gpu": torch.cuda.get_device_name(0),
                      "power_limit_and_max_sm_clock": nvsmi("power.limit,clocks.max.sm")}), flush=True)
    model = build()
    rows = []
    N = a.old
    seq, am = inputs(N, 0)
    vis, vm = inputs(N, 1)
    for tiled in (False, True):  # warm-up of both paths
        run(model, N, tiled, seq, vis, am, vm)
    outs = {}
    for _ in range(a.runs):
        for tiled in (False, True):
            out, ms, peak = run(model, N, tiled, seq, vis, am, vm)
            outs[tiled] = out
            rows.append(row("tiled" if tiled else "all-pairs", N, tiled, ms, peak))
    diff = float((outs[True] - outs[False]).abs().max())
    print(json.dumps({"max_abs_logit_diff_tiled_vs_all_pairs": diff, "N": N}), flush=True)
    del seq, vis, am, vm, outs
    profiles = []
    for N in [int(s) for s in a.sizes.split(",") if s]:
        seq, am = inputs(N, 2)
        vis, vm = inputs(N, 3)
        n = min(N, 512)  # warm-up of every precision at every size: loads each kernel before the timed calls
        for p in precisions:
            run(model, n, True, seq[:n], vis[:n], am[:n], vm[:n], p)
        runs = 1 if N > 2048 and len(precisions) == 1 else a.runs
        for _ in range(runs):
            ref = None
            for p in precisions:
                out, ms, peak = run(model, N, True, seq, vis, am, vm, p)
                d = None
                if p == "bf16":
                    ref = out
                elif ref is not None:
                    d = float((out - ref).abs().max())
                rows.append(row("tiled", N, True, ms, peak, p, d))
                del out
            del ref
        if len(precisions) > 1:
            for p in precisions:
                profiles.append(profile(model, N, seq, vis, am, vm, p))
        del seq, vis, am, vm
    os.environ.pop("UNIVL_EVAL_PRECISION", None)
    print("\n| path | precision | pairs | ms | pairs/s | TFLOP | TFLOP/s | peak GiB |")
    print("|---|---|---|---|---|---|---|---|")
    for r in rows:
        print("| %s | %s | %d x %d | %.1f | %.3g | %.2f | %.1f | %.2f |" % (
            r["path"], r["precision"], r["Nt"], r["Nv"], r["ms"], r["pairs_per_s"], r["tflop"], r["tflop_per_s"],
            r["peak_gib"]))
    if profiles:
        print("\n| precision | pairs | GEMM ms | other ms | GEMM share |\n|---|---|---|---|---|")
        for r in profiles:
            print("| %s | %d x %d | %.1f | %.1f | %.2f |" % (r["precision"], r["Nt"], r["Nv"], r["gemm_ms"],
                                                            r["other_ms"], r["gemm_share"]))


if __name__ == "__main__":
    main()
