"""Time retrieval over large galleries (univl_b200.retrieval) on random bf16 encoder outputs with ragged masks, as
scripts/bench_retrieval_eval.py builds them (W = F = 48, two cross layers, FT-Align model):

  (a) topk:   retrieval.topk_similarity against UniVL._mean_pool_similarity followed by torch.topk, at the --topk sizes
              (Nt x Nv; the dense matrix must fit, and the similarity kernel indexes at most 2^26 entries).  The two
              are alternated; the shortlist's indices must equal torch.topk's wherever no two scores tie.
  (b) pairs:  retrieval.score_pairs on a k-per-query list (--k_list per text row) against the full grid
              (get_similarity_logits) at the --grid size, both under UNIVL_EVAL_LAYOUT=padded and bf16.
  (c) search: retrieval.search(model, model, ..., --k_shortlist, --k) on a gallery too large for the grid (--search).

Per row: ms per call (host clock around a device synchronise, one untimed call first), the torch allocator's peak
above the inputs, and for the shortlist its algorithmic FLOPs 2 Nt Nv H with the achieved fp32 rate against the H100
SXM data-sheet 67 TFLOP/s.  The card's name, power limit and SM clock are read in the same run.  Prints one JSON line
per row.

usage: python scripts/bench_retrieval_search.py [--topk 3500x3500,5000x10000] [--grid 1024] [--k_list 50]
                                               [--search 20000x100000] [--k_shortlist 50] [--k 10]
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

H, W, F, LAYERS = 768, 48, 48, 2
FP32_PEAK = 67e12  # H100 SXM data sheet, dense fp32, 700 W


def nvsmi(query):
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=" + query, "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else None
    except (OSError, subprocess.SubprocessError):
        return None


def build():
    from oracle import synth
    from tests.model_util import build_model
    cfg = synth.task_config(mode="ft_align", batch_size=2, text_layers=1, visual_layers=1, cross_layers=LAYERS,
                            max_words=W, max_frames=F)
    return build_model(cfg, seed=0).eval()


def inputs(N, L, seed):
    """N random rows of encoder output (generated on the device) and ragged prefix masks, lengths in [L/4, L]"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(N, L, H, generator=g, device="cuda").to(torch.bfloat16)
    lens = torch.randint(L // 4, L + 1, (N,), generator=g, device="cuda")
    return x, (torch.arange(L, device="cuda").view(1, L) < lens.view(N, 1)).long()


def timed(fn):
    """-> (result, ms, peak bytes above what was allocated before the call)"""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3
    return out, ms, torch.cuda.max_memory_allocated() - base


def emit(rows, **kw):
    print(json.dumps(kw), flush=True)
    rows.append(kw)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--topk", default="3500x3500,5000x10000")
    ap.add_argument("--grid", type=int, default=1024)
    ap.add_argument("--k_list", type=int, default=50)
    ap.add_argument("--search", default="20000x100000")
    ap.add_argument("--k_shortlist", type=int, default=50)
    ap.add_argument("--k", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_retrieval_search: no CUDA device")
    from univl_b200 import retrieval
    from univl_b200 import runtime as rt
    os.environ["UNIVL_EVAL_LAYOUT"] = "padded"
    os.environ["UNIVL_EVAL_PRECISION"] = "bf16"
    card = {"gpu": torch.cuda.get_device_name(), "power_limit": nvsmi("power.limit"),
            "sm_clock_max": nvsmi("clocks.max.sm"), "sm_clock_now": nvsmi("clocks.sm")}
    print(json.dumps(card), flush=True)
    model = build()
    rows = []

    for size in filter(None, args.topk.split(",")):
        Nt, Nv = (int(x) for x in size.split("x"))
        seq, am = inputs(Nt, W, 2 * Nt)
        vis, vm = inputs(Nv, F, 2 * Nv + 1)
        k = args.k_list

        def dense():
            with torch.no_grad(), rt.use_model(model, model._device()):
                sim = model._mean_pool_similarity(seq.view(-1, H), vis.view(-1, H), am, vm)
                return torch.topk(sim, k, dim=1)

        def shortlist():
            return retrieval.topk_similarity(model, seq, vis, am, vm, k)
        dense(), shortlist()  # warm-up
        res = {}
        for name, fn in (("dense+torch.topk", dense), ("topk_similarity", shortlist)) * 2:
            (_, idx), ms, peak = timed(fn)
            res[name] = idx
            fl = 2.0 * Nt * Nv * H
            emit(rows, part="topk", variant=name, Nt=Nt, Nv=Nv, k=k, ms=round(ms, 2), peak_gib=round(peak / 2 ** 30, 3),
                 gflop=round(fl / 1e9, 1), tflop_per_s=round(fl / ms / 1e9, 2),
                 share_of_fp32_peak=round(fl / ms / 1e9 / (FP32_PEAK / 1e12), 3))
        same = float((res["dense+torch.topk"].long() == res["topk_similarity"]).float().mean())
        emit(rows, part="topk", Nt=Nt, Nv=Nv, index_agreement_with_torch_topk=same)
        del seq, vis, am, vm

    N = args.grid
    seq, am = inputs(N, W, 10)
    vis, vm = inputs(N, F, 11)
    ti = torch.arange(N, device="cuda").repeat_interleave(args.k_list)
    vi = torch.randint(0, N, (N * args.k_list,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    with torch.no_grad():
        retrieval.score_pairs(model, seq[:8], vis[:8], am[:8], vm[:8], ti[:8] % 8, vi[:8] % 8)
        grid, ms, peak = timed(lambda: model.get_similarity_logits(seq, vis, am, vm))
        emit(rows, part="pairs", variant="grid", Nt=N, Nv=N, pairs=N * N, ms=round(ms, 1),
             pairs_per_s=round(N * N / ms * 1e3), peak_gib=round(peak / 2 ** 30, 3))
        got, ms, peak = timed(lambda: retrieval.score_pairs(model, seq, vis, am, vm, ti, vi))
        emit(rows, part="pairs", variant="score_pairs", Nt=N, Nv=N, pairs=ti.numel(), ms=round(ms, 1),
             pairs_per_s=round(ti.numel() / ms * 1e3), peak_gib=round(peak / 2 ** 30, 3),
             equal_to_grid=bool(torch.equal(got, grid[ti, vi])))
    del seq, vis, am, vm, grid

    Nt, Nv = (int(x) for x in args.search.split("x"))
    seq, am = inputs(Nt, W, 20)
    vis, vm = inputs(Nv, F, 21)
    retrieval.search(model, model, seq[:64], vis[:4096], am[:64], vm[:4096], args.k_shortlist, args.k)
    (s, i), ms, peak = timed(lambda: retrieval.search(model, model, seq, vis, am, vm, args.k_shortlist, args.k))
    (_, _), ms_short, _ = timed(lambda: retrieval.topk_similarity(model, seq, vis, am, vm, args.k_shortlist))
    fl = 2.0 * Nt * Nv * H
    emit(rows, part="search", Nt=Nt, Nv=Nv, k_shortlist=args.k_shortlist, k=args.k, ms=round(ms, 1),
         shortlist_ms=round(ms_short, 1), rerank_pairs=Nt * args.k_shortlist, peak_gib=round(peak / 2 ** 30, 3),
         shortlist_tflop_per_s=round(fl / ms_short / 1e9, 2),
         dense_fp32_matrix_gib=round(Nt * Nv * 4 / 2 ** 30, 1), **card)


if __name__ == "__main__":
    main()
