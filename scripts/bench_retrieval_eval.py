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

--layout padded,packed alternates the tiled path's layouts (UNIVL_EVAL_LAYOUT) within every run as well, the pairs
computed at W + F tokens or on their valid tokens alone, and --valid picks the valid-length distributions, each run
in turn: "uniform" (default; text and clip lengths uniform in [L/4, L]) and "short" (text 8-20 tokens, clips 12-30
frames).  Rows then also give the packed-token fraction (valid pair tokens / padded pair tokens), the max |logit
difference| of packed against padded at the same precision, and a second rate, tflop_per_s_packed: the FLOPs of the
packed tokens actually computed (same formula, S the pair's valid tokens) per second.  tflop_per_s stays the
algorithmic count over padded tokens for every layout.

FLOPs (multiply-add = 2) per pair at S = W + F, H = 768, I = 3072, L cross layers, the last one token-0 only:
  (L-1) S (8H^2 + 4HI + 4SH)  +  S 4H^2 (last layer K/V)  +  2H^2 + 4SH + 2H^2 + 4HI (last layer, token 0)  +  2H^2
  (pooler); (b) does S 6H^2 less per pair (first layer Q/K/V) and (Nt W + Nv F) 6H^2 once per call.

usage: python scripts/bench_retrieval_eval.py [--old 128] [--sizes 1024,3500] [--runs 3] [--precision bf16,fp8]
                                             [--layout padded,packed] [--valid uniform,short]
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


def flops_packed(am, vm):
    """flops(tiled=True) with every pair at its valid length S_ij = len_t(i) + len_v(j): sums of S and S^2 over pairs"""
    lt, lv = am.sum(1).double().cpu(), vm.sum(1).double().cpu()
    Nt, Nv = lt.numel(), lv.numel()
    T = float(Nv * lt.sum() + Nt * lv.sum())                                         # sum of S
    Q = float(Nv * (lt * lt).sum() + 2 * lt.sum() * lv.sum() + Nt * (lv * lv).sum())  # sum of S^2
    return ((LAYERS - 1) * (T * (8 * H * H + 4 * H * I) + 4 * Q * H) + T * 4 * H * H
            + Nt * Nv * (6 * H * H + 4 * H * I) + 4 * T * H - T * 6 * H * H + (Nt * W + Nv * F) * 6 * H * H)


# valid-length range per role (text rows, video rows), inclusive; None: uniform in [L/4, L] for a row of L tokens
VALID = {"uniform": None, "short": {"text": (8, 20), "video": (12, 30)}}


def build():
    from oracle import synth
    from tests.model_util import build_model
    cfg = synth.task_config(mode="ft_align", batch_size=2, text_layers=1, visual_layers=1, cross_layers=LAYERS,
                            max_words=W, max_frames=F)
    return build_model(cfg, seed=0).eval()


def inputs(N, seed, valid="uniform"):
    """N random rows of encoder output and their mask: text rows (W tokens) for an even seed, video rows (F) for odd"""
    g = torch.Generator().manual_seed(seed)
    role = "text" if seed % 2 == 0 else "video"
    L = W if role == "text" else F
    x = torch.randn(N, L, H, generator=g).to(torch.bfloat16).cuda()
    lo, hi = VALID[valid][role] if VALID[valid] else (L // 4, L)
    lens = torch.randint(lo, hi + 1, (N,), generator=g)
    return x, (torch.arange(L).view(1, L) < lens.view(N, 1)).long().cuda()


def run(model, N, tiled, seq, vis, am, vm, precision="bf16", layout="padded"):
    from univl_b200 import runtime as rt
    os.environ["UNIVL_EVAL_PRECISION"] = precision
    os.environ["UNIVL_EVAL_LAYOUT"] = layout
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


def profile(model, N, seq, vis, am, vm, precision, layout="padded", valid="uniform"):
    """GPU time of one tiled call, split into GEMM kernels, attention kernels and everything else"""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity
    with torch.profiler.profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(model, N, True, seq, vis, am, vm, precision, layout)
    gemm = attn = other = 0.0
    for e in prof.key_averages():
        if e.device_type != DeviceType.CUDA:
            continue
        if "gemm" in e.key:
            gemm += e.self_device_time_total
        elif "attention" in e.key:
            attn += e.self_device_time_total
        else:
            other += e.self_device_time_total
    r = dict(profile="tiled", precision=precision, layout=layout, valid=valid, Nt=N, Nv=N,
             gemm_ms=round(gemm / 1e3, 1), attention_ms=round(attn / 1e3, 1), other_ms=round(other / 1e3, 1),
             gemm_share=round(gemm / max(gemm + attn + other, 1e-9), 3))
    print(json.dumps(r), flush=True)
    return r


def row(name, N, tiled, ms, peak, precision="bf16", dlogit=None, layout="padded", valid="uniform", masks=None,
        dpacked=None):
    from univl_b200.modules import modeling
    f = flops(N, N, tiled)
    r = dict(path=name, precision=precision, layout=layout, valid=valid, Nt=N, Nv=N, W=W, F=F, cross_layers=LAYERS,
             ms=round(ms, 2), pairs_per_s=round(N * N / ms * 1e3), tflop=round(f / 1e12, 2),
             tflop_per_s=round(f / ms / 1e9, 1), peak_gib=round(peak / 2 ** 30, 3))
    if masks is not None:
        am, vm = masks
        r["packed_fraction"] = round(float(N * (am.sum() + vm.sum())) / (N * N * (W + F)), 4)
        if layout == "packed":
            r["tflop_per_s_packed"] = round(flops_packed(am, vm) / ms / 1e9, 1)
    if dpacked is not None:
        r["max_abs_dlogit_vs_padded"] = dpacked
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
    ap.add_argument("--layout", default="padded", help="comma-separated eval layouts of the tiled path: padded,packed")
    ap.add_argument("--valid", default="uniform", help="comma-separated valid-length distributions: uniform,short")
    a = ap.parse_args()
    precisions = [p for p in a.precision.split(",") if p]
    layouts = [x for x in a.layout.split(",") if x]
    if "padded" not in layouts:
        layouts.insert(0, "padded")  # the reference result of the packed logit differences
    valids = [x for x in a.valid.split(",") if x]
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
    for valid in valids:
        for N in [int(s) for s in a.sizes.split(",") if s]:
            seq, am = inputs(N, 2, valid)
            vis, vm = inputs(N, 3, valid)
            n = min(N, 512)  # warm-up of every variant at every size: loads each kernel before the timed calls
            for lay in layouts:
                for p in precisions:
                    run(model, n, True, seq[:n], vis[:n], am[:n], vm[:n], p, lay)
            runs = 1 if N > 2048 and len(precisions) * len(layouts) == 1 else a.runs
            for _ in range(runs):
                ref = None
                padded = {}
                for lay in layouts:
                    for p in precisions:
                        out, ms, peak = run(model, N, True, seq, vis, am, vm, p, lay)
                        d = dp = None
                        if lay == "padded":
                            padded[p] = out
                        elif p in padded:
                            dp = float((out - padded[p]).abs().max())
                        if p == "bf16" and lay == "padded":
                            ref = out
                        elif p != "bf16" and ref is not None:
                            d = float((out - ref).abs().max())
                        rows.append(row("tiled", N, True, ms, peak, p, d, lay, valid, (am, vm), dp))
                        del out
                del ref, padded
            if len(precisions) * len(layouts) > 1:
                for lay in layouts:
                    for p in precisions:
                        profiles.append(profile(model, N, seq, vis, am, vm, p, lay, valid))
            del seq, vis, am, vm
    os.environ.pop("UNIVL_EVAL_PRECISION", None)
    os.environ.pop("UNIVL_EVAL_LAYOUT", None)
    print("\n| path | layout | valid | precision | pairs | ms | pairs/s | packed frac | TFLOP | TFLOP/s (padded) "
          "| TFLOP/s (packed) | max dlogit vs padded | peak GiB |")
    print("|---|---|---|---|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        print("| %s | %s | %s | %s | %d x %d | %.1f | %.3g | %s | %.2f | %.1f | %s | %s | %.2f |" % (
            r["path"], r["layout"], r["valid"], r["precision"], r["Nt"], r["Nv"], r["ms"], r["pairs_per_s"],
            r.get("packed_fraction", "-"), r["tflop"], r["tflop_per_s"], r.get("tflop_per_s_packed", "-"),
            r.get("max_abs_dlogit_vs_padded", "-"), r["peak_gib"]))
    if profiles:
        print("\n| layout | valid | precision | pairs | GEMM ms | attention ms | other ms | GEMM share |\n"
              "|---|---|---|---|---|---|---|---|")
        for r in profiles:
            print("| %s | %s | %s | %d x %d | %.1f | %.1f | %.1f | %.2f |" % (
                r["layout"], r["valid"], r["precision"], r["Nt"], r["Nv"], r["gemm_ms"], r["attention_ms"],
                r["other_ms"], r["gemm_share"]))


if __name__ == "__main__":
    main()
