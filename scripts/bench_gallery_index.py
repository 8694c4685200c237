"""Gallery indexing on valid tokens (univl_b200.retrieval.embed_texts / embed_videos / topk) against the padded
encoders, on one GPU.

Encode: N clips at F frames and N queries at W tokens with the FT-Joint encoders (12 text layers, 6 visual layers),
under the length mixes --valid ("uniform": lengths uniform in [L/4, L]; "short": text 8-20 tokens, clips 12-30 frames,
as scripts/bench_retrieval_eval.py; "full": every token valid).  The padded path is what get_sequence_visual_output
computes followed by MeanPoolFn (NormalizeVideo + visual encoder, or the text encoder, at every padded token), run in
chunks of EMBED_TOKENS padded tokens so that its memory is bounded too; the packed path is embed_videos /
embed_texts.  The two run alternately in one process, --reps times after one warm-up each; the best time is reported.
TFLOP/s counts the dense and attention FLOPs of the tokens each path computes (packed: the valid ones).

Search: --queries stored query vectors against --gallery stored clip vectors (comma-separated sizes) with k = --k
through retrieval.topk, and topk_similarity on --seq-gallery clips of bf16 sequence outputs for comparison; the best
of --reps runs after one warm-up, as for encoding.

The card's name, power limit and SM clock are read in the same process and printed with the results.  One JSON line
per measurement.
  python scripts/bench_gallery_index.py [--n 100000] [--valid uniform,short,full] [--reps 2] [--queries 5000]
                                        [--gallery 100000,1000000] [--seq-gallery 100000] [--k 50]
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

H, I, W, F, D = 768, 3072, 48, 48, 1024
TEXT_LAYERS, VISUAL_LAYERS = 12, 6
VALID = {"uniform": None, "short": {"text": (8, 20), "video": (12, 30)}, "full": "full"}


def nvsmi(query):
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=" + query, "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else None
    except (OSError, subprocess.SubprocessError):
        return None


def encoder_flops(lens, layers, proj_in=0):
    """dense FLOPs of `layers` encoder layers over sequences of the given lengths (+ attention's 4 S^2 H per layer),
    plus the input projection (proj_in -> H) per token"""
    lens = lens.double()
    T, Q = float(lens.sum()), float((lens * lens).sum())
    return layers * (T * (8 * H * H + 4 * H * I) + 4 * Q * H) + T * 2 * proj_in * H


def lengths(N, L, role, valid, g):
    spec = VALID[valid]
    if spec == "full":
        return torch.full((N,), L, dtype=torch.long)
    lo, hi = spec[role] if spec else (L // 4, L)
    return torch.randint(lo, hi + 1, (N,), generator=g)


def build():
    from oracle import synth
    from tests.model_util import build_model
    cfg = synth.task_config(mode="ft_joint", batch_size=2, text_layers=TEXT_LAYERS, visual_layers=VISUAL_LAYERS,
                            max_words=W, max_frames=F)
    return build_model(cfg, seed=0).eval()


def padded_texts(model, ids, am, budget):
    from univl_b200 import ops
    from univl_b200 import runtime as rt
    out = torch.empty((ids.shape[0], H), dtype=torch.float32, device=ids.device)
    rows = max(1, budget // W)
    with rt.use_model(model, model._device()):
        for a in range(0, ids.shape[0], rows):
            b = min(ids.shape[0], a + rows)
            seq = model.bert.encode(ids[a:b], torch.zeros_like(ids[a:b]), am[a:b])
            out[a:b] = ops.MeanPoolFn.apply(seq, am[a:b], b - a, W, True, False, True)
    return out


def padded_videos(model, video, vm, budget):
    from univl_b200 import ops
    from univl_b200 import runtime as rt
    out = torch.empty((video.shape[0], H), dtype=torch.float32, device=video.device)
    rows = max(1, budget // F)
    with rt.use_model(model, model._device()):
        for a in range(0, video.shape[0], rows):
            b = min(video.shape[0], a + rows)
            vis = model.visual.encode(model.normalize_video(video[a:b]), vm[a:b])
            out[a:b] = ops.MeanPoolFn.apply(vis, vm[a:b], b - a, F, False, True, True)
    return out


def timed(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0, torch.cuda.max_memory_allocated() - base


def best_of(fn, reps):
    """(seconds, peak bytes) of the fastest of `reps` runs after one warm-up"""
    runs = [timed(fn)[1:] for _ in range(reps + 1)][1:]
    return min(runs)


def encode(model, N, valid, reps, card):
    from univl_b200 import retrieval
    from univl_b200.modules import modeling
    g = torch.Generator().manual_seed(7)
    lt, lv = lengths(N, W, "text", valid, g), lengths(N, F, "video", valid, g)
    am = (torch.arange(W)[None] < lt[:, None]).long().cuda()
    vm = (torch.arange(F)[None] < lv[:, None]).long().cuda()
    ids = torch.randint(1000, 30000, (N, W), generator=g).cuda()
    video = torch.empty((N, F, D), dtype=torch.float32, device="cuda").normal_(generator=torch.Generator(
        device="cuda").manual_seed(8))
    budget = modeling.EMBED_TOKENS
    runs = {
        ("video", "padded"): lambda: padded_videos(model, video, vm, budget),
        ("video", "packed"): lambda: retrieval.embed_videos(model, video, vm),
        ("text", "padded"): lambda: padded_texts(model, ids, am, budget),
        ("text", "packed"): lambda: retrieval.embed_texts(model, ids, am),
    }
    best, outs = {}, {}
    with torch.no_grad():
        for rep in range(reps + 1):
            for key, fn in runs.items():
                out, s, peak = timed(fn)
                outs[key] = out
                if rep > 0 and (key not in best or s < best[key][0]):
                    best[key] = (s, peak)
    for role, lens, L, layers, proj in (("video", lv, F, VISUAL_LAYERS, D), ("text", lt, W, TEXT_LAYERS, 0)):
        pad, pk = outs[(role, "padded")], outs[(role, "packed")]
        fin = torch.isfinite(pad).all(1) & torch.isfinite(pk).all(1)
        diff = float((pad[fin] - pk[fin]).abs().max())
        for layout, computed in (("padded", torch.full_like(lens, L)), ("packed", lens)):
            s, peak = best[(role, layout)]
            print(json.dumps(dict(
                bench="encode", role=role, layout=layout, valid=valid, n=N, seconds=round(s, 4),
                rows_per_s=round(N / s), packed_fraction=round(float(lens.sum()) / (N * L), 3),
                tflops=round(encoder_flops(computed, layers, proj) / s / 1e12, 1),
                max_abs_diff_vs_padded=diff, peak_gib=round(peak / 2 ** 30, 2), **card)), flush=True)


def search(model, queries, galleries, seq_gallery, k, reps, card):
    from univl_b200 import retrieval
    g = torch.Generator(device="cuda").manual_seed(9)

    def unit(n):
        x = torch.empty((n, H), dtype=torch.float32, device="cuda").normal_(generator=g)
        return x / x.norm(dim=1, keepdim=True)
    q = unit(queries)
    for n in galleries:
        gal = unit(n)
        sec, peak = best_of(lambda: retrieval.topk(q, gal, k), reps)
        print(json.dumps(dict(bench="search", stored="vectors", queries=queries, gallery=n, k=k,
                              seconds=round(sec, 4), peak_gib=round(peak / 2 ** 30, 2),
                              tflops_fp32=round(2.0 * queries * n * H / sec / 1e12, 1), **card)), flush=True)
        del gal
    if seq_gallery:
        seq = torch.empty((queries, W, H), dtype=torch.bfloat16, device="cuda").normal_(generator=g)
        vis = torch.empty((seq_gallery, F, H), dtype=torch.bfloat16, device="cuda").normal_(generator=g)
        am = torch.ones((queries, W), dtype=torch.long, device="cuda")
        vm = torch.ones((seq_gallery, F), dtype=torch.long, device="cuda")
        with torch.no_grad():
            sec, peak = best_of(lambda: retrieval.topk_similarity(model, seq, vis, am, vm, k), reps)
        print(json.dumps(dict(bench="search", stored="sequence_outputs", queries=queries, gallery=seq_gallery, k=k,
                              seconds=round(sec, 4), peak_gib=round(peak / 2 ** 30, 2), **card)), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--n", type=int, default=100000)
    ap.add_argument("--valid", default="uniform,short,full")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--queries", type=int, default=5000)
    ap.add_argument("--gallery", default="100000,1000000")
    ap.add_argument("--seq-gallery", type=int, default=100000)
    ap.add_argument("--k", type=int, default=50)
    ap.add_argument("--skip-encode", action="store_true")
    args = ap.parse_args()
    mixes = [v for v in args.valid.split(",") if v]
    for v in mixes:
        if v not in VALID:
            ap.error("unknown --valid %r (one of %s)" % (v, ",".join(VALID)))
    if not torch.cuda.is_available():
        sys.exit("bench_gallery_index.py needs a CUDA device")
    card = dict(gpu=nvsmi("name"), power_limit=nvsmi("power.limit"), sm_clock_max=nvsmi("clocks.max.sm"),
                sm_clock=nvsmi("clocks.sm"))
    model = build()
    if not args.skip_encode:
        for v in mixes:
            encode(model, args.n, v, args.reps, card)
    search(model, args.queries, [int(x) for x in args.gallery.split(",") if x], args.seq_gallery, args.k,
           args.reps, card)
    card["sm_clock_after"] = nvsmi("clocks.sm")
    print(json.dumps(dict(bench="card", **card)), flush=True)


if __name__ == "__main__":
    main()
