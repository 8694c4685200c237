"""Ground-truth ranks at gallery scale (univl_b200.retrieval.ranks), on one GPU: speed against topk, and the recall the
shortlist search had not measured.

Speed: retrieval.ranks against retrieval.topk at k = 10 on the same stored vectors (H = 768, unit-norm, seeded):
--queries queries against each of --gallery rows, text-to-video and video-to-text, and --videos videos with --captions
captions each (video-to-text with that many positives per query, and text-to-video with that many queries per
video).  Each is timed with CUDA events over --reps calls after one warm-up; TFLOP/s counts 2 Nq Ng H.  At
--dense-gallery rows, where the [Nq, Ng] fp32 matrix fits, the dense path (ops.SimMatmulFn + ranks_from_scores) is
timed too, and all three paths are checked to agree.

Quality: the synthetic matched-pair task and training recipe of scripts/eval_fp8_quality.py (this is not YouCookII or
MSRVTT data).  It trains two reduced models: an FT-Joint model, which ranks by the mean-pooled similarity, and the
FT-Align cross encoder that script trains.  Then it reports on the held-out pairs:
  - the FT-Joint model's text-to-video and video-to-text rank_metrics from stored vectors (embed_texts, embed_videos);
  - the FT-Align model's own text-to-video rank_metrics from its dense logits (ranks_from_scores);
  - the fraction of texts whose FT-Align top-1 video (the argmax of its dense logits) falls inside the FT-Joint
    shortlist of 10 / 50 / 100: ranks(texts, videos, query_labels=top1) < K.

The card's name, power limit and SM clock are read in the same process.  One JSON line per measurement.
  python scripts/bench_retrieval_ranks.py [--queries 5000] [--gallery 100000,1000000] [--videos 1000] [--captions 20]
                                          [--dense-gallery 100000] [--reps 3] [--skip-quality] [--skip-speed]
                                          [eval_fp8_quality.py's task and training options]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from scripts import eval_fp8_quality as task  # noqa: E402
from scripts.bench_gallery_index import nvsmi  # noqa: E402

H, K = 768, 10


def unit(n, g):
    x = torch.empty((n, H), dtype=torch.float32, device="cuda").normal_(generator=g)
    return x / x.norm(dim=1, keepdim=True)


def time_s(fn, reps):
    """mean seconds per call over `reps` calls after one warm-up, by CUDA events"""
    fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / 1e3 / reps


def speed_case(name, q, g, ql, gl, reps, card, dense=False):
    from univl_b200 import ops
    from univl_b200 import retrieval
    Nq, Ng = q.shape[0], g.shape[0]
    flops = 2.0 * Nq * Ng * H
    r = retrieval.ranks(q, g, ql, gl)
    _, idx = retrieval.topk(q, g, K)
    # rank < K exactly when a positive is in the top K, at position rank
    glab = torch.arange(Ng, device="cuda") if gl is None else gl.long()
    qlab = torch.arange(Nq, device="cuda") if ql is None else ql.long()
    hit = glab[idx] == qlab[:, None]
    first = torch.where(hit.any(1), hit.int().argmax(1), torch.full_like(r, K))
    consistent = bool(torch.equal(torch.minimum(r, torch.full_like(r, K)), first))
    rows = {"ranks": time_s(lambda: retrieval.ranks(q, g, ql, gl), reps),
            "topk_k10": time_s(lambda: retrieval.topk(q, g, K), reps)}
    if dense:
        rows["dense"] = time_s(lambda: retrieval.ranks_from_scores(ops.SimMatmulFn.apply(q, g, 1), ql, gl), reps)
        consistent &= bool(torch.equal(retrieval.ranks_from_scores(ops.SimMatmulFn.apply(q, g, 1), ql, gl), r))
    for path, sec in rows.items():
        print(json.dumps(dict(bench="speed", case=name, path=path, queries=Nq, gallery=Ng, H=H, seconds=round(sec, 4),
                              tflops_fp32=round(flops / sec / 1e12, 1), ranks_agree=consistent,
                              median_rank=int(r.median()), **card)), flush=True)


def speed(a, card):
    g = torch.Generator(device="cuda").manual_seed(9)
    texts = unit(a.queries, g)
    with torch.no_grad():
        for n in a.gallery:
            videos = unit(n, g)
            speed_case("t2v", texts, videos, None, None, a.reps, card, dense=n == a.dense_gallery)
            speed_case("v2t", videos[:a.queries], unit(n, g), None, None, a.reps, card)
            del videos
            torch.cuda.empty_cache()
        # many captions per video: captions near their video
        videos = unit(a.videos, g)
        owner = torch.arange(a.videos * a.captions, device="cuda") // a.captions
        caps = videos[owner] + 0.1 * unit(owner.numel(), g)
        caps = caps / caps.norm(dim=1, keepdim=True)
        speed_case("v2t_%d_captions" % a.captions, videos, caps, None, owner, a.reps, card, dense=True)
        speed_case("t2v_%d_captions" % a.captions, caps, videos, owner, None, a.reps, card, dense=True)


def quality(a, card):
    from univl_b200 import retrieval
    torch.manual_seed(a.seed)
    sample = task.make_task(a.vocab, a.noise, a.seed + 1)
    held_out = sample(a.eval, seed=10 ** 6)
    print(json.dumps({"bench": "quality_task", "task": "synthetic matched pairs (scripts/eval_fp8_quality.py)",
                      "options": vars(a), "chance_R1": 1.0 / a.eval, **card}), flush=True)

    def vectors(model, d):
        model.eval()
        with torch.no_grad():
            t = retrieval.embed_texts(model, d["input_ids"], d["attention_mask"], d["token_type_ids"])
            v = retrieval.embed_videos(model, d["video"], d["video_mask"])
        return t, v

    def joint_eval(model, d):
        m = retrieval.rank_metrics(retrieval.ranks(*vectors(model, d)))
        return {"R@1": round(100 * m["R1"], 2), "MR": m["MR"]}

    joint, joint_steps = task.train(a, "ft_joint", sample, held_out, joint_eval)
    t, v = vectors(joint, held_out)
    out = {"bench": "quality", "ft_joint_steps": joint_steps,
           "ft_joint_t2v": retrieval.rank_metrics(retrieval.ranks(t, v)),
           "ft_joint_v2t": retrieval.rank_metrics(retrieval.ranks(v, t))}
    del joint
    align, align_steps = task.train(a, "ft_align", sample, held_out,
                                    lambda m, d: task.metrics(task.logits(m, d, "bf16")))
    logits = task.logits(align, held_out, "bf16").contiguous()
    top1 = logits.argmax(1)
    inside = retrieval.ranks(t, v, query_labels=top1)
    out.update({"ft_align_steps": align_steps,
                "ft_align_t2v": retrieval.rank_metrics(retrieval.ranks_from_scores(logits)),
                "ft_align_top1_is_true_video": float((top1 == torch.arange(a.eval, device="cuda")).float().mean())})
    for k in (10, 50, 100):
        out["align_top1_in_joint_shortlist_%d" % k] = float((inside < k).float().mean())
    print(json.dumps(dict(out, **card)), flush=True)


def main():
    ap = task.arguments(argparse.ArgumentParser(description=__doc__.split("\n")[0]))
    ap.add_argument("--queries", type=int, default=5000)
    ap.add_argument("--gallery", default="100000,1000000")
    ap.add_argument("--videos", type=int, default=1000)
    ap.add_argument("--captions", type=int, default=20)
    ap.add_argument("--dense-gallery", type=int, default=100000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--skip-speed", action="store_true")
    ap.add_argument("--skip-quality", action="store_true")
    a = ap.parse_args()
    a.gallery = [int(x) for x in a.gallery.split(",") if x]
    if not torch.cuda.is_available():
        sys.exit("bench_retrieval_ranks.py needs a CUDA device")
    card = dict(gpu=nvsmi("name"), power_limit=nvsmi("power.limit"), sm_clock_max=nvsmi("clocks.max.sm"),
                sm_clock=nvsmi("clocks.sm"))
    if not a.skip_speed:
        speed(a, card)
    if not a.skip_quality:
        quality(a, card)
    card["sm_clock_after"] = nvsmi("clocks.sm")
    print(json.dumps(dict(bench="card", **card)), flush=True)


if __name__ == "__main__":
    main()
