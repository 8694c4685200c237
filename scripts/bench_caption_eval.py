"""Time the caption driver's beam-search evaluation (the reference's main_task_caption.eval_epoch, run unmodified
through univl_b200.launcher) on synthetic batches, in three configurations alternated in one process:

  off        UNIVL_DECODE_CACHE=off: every decoder_caption call computes its full prefix
  cache      UNIVL_DECODE_CACHE=prefix with the checkout's Beam (one device read per token per hypothesis)
  cache+host UNIVL_DECODE_CACHE=prefix with univl_b200.modules.beam.Beam (hypotheses on the host)

and, for comparison, univl_b200.caption.beam_search and univl_b200.caption.GraphBeamSearch ("graph": the loop on the
device, replayed as CUDA graphs; one searcher per cap, so its graphs are captured in the warm-up) on the same inputs.  A randomly initialised model never ranks [SEP]
first, so the decode cap (the driver's --max_words loop bound) fixes the number of steps.  Reports ms per batch and
the peak of torch allocations, with the card's name and power limit read in the same run; --profile adds a
torch.profiler run of one batch per configuration: the summed time of its device events, and the rest of the profiled
wall time (host gaps; the profiler itself slows the host, so these runs are not the timed ones).

    python scripts/bench_caption_eval.py --shape youcook --cap 20 --batches 2
"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

# the README's settings: YouCookII 12 text / 6 visual / 2 cross / 3 decoder layers, W = 128, F = 96; MSRVTT W = F = 48
SHAPES = {"youcook": dict(W=128, F=96), "msrvtt": dict(W=48, F=48), "tiny": dict(W=16, F=16)}
CONFIGS = ("off", "cache", "cache+host", "beam_search", "graph")
_SEARCHERS = {}


class FakeTokenizer(object):
    """the four special tokens of bert-base-uncased; every other id prints as w<id>"""
    vocab = {"[PAD]": 0, "[UNK]": 100, "[CLS]": 101, "[SEP]": 102}
    _names = {v: k for k, v in vocab.items()}

    def convert_ids_to_tokens(self, ids):
        return [self._names.get(int(i), "w%d" % int(i)) for i in ids]


class FakeNLGEval(object):
    """captures the lists eval_epoch scores; every metric reads 0"""

    def __init__(self):
        self.calls = []

    def compute_metrics(self, ref_list, hyp_list):
        self.calls.append((ref_list, list(hyp_list)))
        return {k: 0.0 for k in ("Bleu_1", "Bleu_2", "Bleu_3", "Bleu_4", "METEOR", "ROUGE_L", "CIDEr")}


def load_driver(root, log_dir):
    """the reference's main_task_caption module, imported through the launcher's shims (it joins an NCCL group of one
    at import) -> (module, the checkout's Beam class)"""
    from univl_b200 import launcher
    launcher.prepare(os.path.join(root, "main_task_caption.py"))
    drv = importlib.import_module("main_task_caption")
    import util
    drv.logger = util.get_logger(os.path.join(log_dir, "log.txt"))
    spec = importlib.util.spec_from_file_location("_checkout_beam", os.path.join(root, "modules", "beam.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return drv, mod.Beam


def make_loader(cfg, n, batch_size, seed):
    """batches in the order eval_epoch unpacks them (input_ids, input_mask, segment_ids, video, video_mask, masked text,
    token labels, masked video, video label index, caption input ids, decoder mask, caption output ids)"""
    from oracle import synth
    b = synth.make_batch(cfg, seed=seed, b=n)
    ids = b["input_ids"]
    cap_in = b.get("input_caption_ids", ids)
    items = [ids, b["attention_mask"], b["token_type_ids"], b["video"], b["video_mask"], ids, torch.full_like(ids, -1),
             b["video"], torch.full_like(b["video_mask"], -1), cap_in, b.get("decoder_mask", torch.ones_like(ids)),
             b.get("output_caption_ids", ids)]
    data = torch.utils.data.TensorDataset(*items)
    return torch.utils.data.DataLoader(data, batch_size=batch_size, shuffle=False)


def build(shape, layers, batch_size, seed=0):
    from oracle import synth
    from tests.model_util import build_model
    W, F = SHAPES[shape]["W"], SHAPES[shape]["F"]
    t, v, c, d = layers
    cfg = synth.task_config(mode="caption", batch_size=batch_size, text_layers=t, visual_layers=v, cross_layers=c,
                            decoder_layers=d, max_words=W, max_frames=F)
    model = build_model(cfg, seed=seed)
    model.eval()
    return cfg, model


def run_config(name, drv, model, loader, cap, out_dir, ref_beam, host_beam):
    """-> hypotheses (list of strings) of one pass over the loader"""
    args = argparse.Namespace(max_words=cap, output_dir=out_dir, datatype="youcook")
    device = torch.device("cuda", 0)
    if name in ("beam_search", "graph"):
        from univl_b200.caption import GraphBeamSearch, beam_search
        if name == "graph":
            if cap not in _SEARCHERS:
                _SEARCHERS[cap] = GraphBeamSearch(model, n_beam=5, max_words=cap)
            search = _SEARCHERS[cap]
        else:
            search = lambda seq, vis, am, vm: beam_search(model, seq, vis, am, vm, cap, n_beam=5)
        hyps = []
        os.environ["UNIVL_DECODE_CACHE"] = "off"
        for batch in loader:
            batch = [x.to(device) for x in batch]
            with torch.no_grad():
                seq, vis = model.get_sequence_visual_output(batch[0], batch[2], batch[1], batch[3], batch[4])
                h, _ = search(seq, vis, batch[1].view(seq.shape[0], -1), batch[4].view(seq.shape[0], -1))
            hyps += [" ".join(map(str, x)) for x in h]
        return hyps
    os.environ["UNIVL_DECODE_CACHE"] = "off" if name == "off" else "prefix"
    drv.Beam = host_beam if name == "cache+host" else ref_beam
    nlg = FakeNLGEval()
    # the driver passes a uint8 decoder mask; the package's attention masks are int64
    real = model.decoder_caption
    model.decoder_caption = lambda *a, **k: real(*a[:6], a[6].long(), *a[7:], **k)
    try:
        drv.eval_epoch(args, model, loader, FakeTokenizer(), device, 1, nlgEvalObj=nlg)
    finally:
        del model.decoder_caption
    return nlg.calls[-1][1]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", choices=sorted(SHAPES), default="youcook")
    ap.add_argument("--layers", default="12,6,2,3", help="text,visual,cross,decoder layers")
    ap.add_argument("--batch-size-val", type=int, default=64)
    ap.add_argument("--cap", type=int, default=20, help="decode steps (the driver's --max_words)")
    ap.add_argument("--batches", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=1, help="alternating rounds over the configurations")
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--profile", default="", help="directory for one torch.profiler trace summary per configuration")
    ap.add_argument("--out", default="", help="write the JSON result here as well")
    a = ap.parse_args()
    from oracle import build_ref
    root = build_ref.ref_root()
    if root is None:
        sys.exit("the reference checkout is not staged (python oracle/build_ref.py)")
    tmp = tempfile.mkdtemp(prefix="univl_caption_bench_")
    drv, ref_beam = load_driver(root, tmp)
    from univl_b200.modules.beam import Beam as host_beam
    layers = tuple(int(x) for x in a.layers.split(","))
    cfg, model = build(a.shape, layers, a.batch_size_val)
    loader = make_loader(cfg, a.batches * a.batch_size_val, a.batch_size_val, seed=5)
    configs = a.configs.split(",")
    for name in configs:  # warm-up: one batch of every configuration (graph: at the timed cap, which captures it)
        run_config(name, drv, model, make_loader(cfg, a.batch_size_val, a.batch_size_val, 6),
                   a.cap if name == "graph" else min(a.cap, 3), tmp, ref_beam, host_beam)
    times = {n: [] for n in configs}
    peaks, hyps = {}, {}
    for _ in range(a.repeats):
        for name in configs:
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            t0 = time.perf_counter()
            hyps[name] = run_config(name, drv, model, loader, a.cap, tmp, ref_beam, host_beam)
            torch.cuda.synchronize()
            times[name].append((time.perf_counter() - t0) * 1e3 / a.batches)
            peaks[name] = torch.cuda.max_memory_allocated() / 2 ** 30
    prof = {}
    if a.profile:
        from torch.autograd import DeviceType
        from torch.profiler import ProfilerActivity, profile
        os.makedirs(a.profile, exist_ok=True)
        one = make_loader(cfg, a.batch_size_val, a.batch_size_val, seed=5)
        for name in configs:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as p:
                run_config(name, drv, model, one, a.cap, tmp, ref_beam, host_beam)
                torch.cuda.synchronize()
            wall = (time.perf_counter() - t0) * 1e3
            # device-side events only (kernels, memcpy, memset), each counted once: operator rows also carry device
            # time totals, so summing the key averages would count every kernel twice
            gpu = sum(e.time_range.elapsed_us() for e in p.events() if e.device_type == DeviceType.CUDA) / 1e3
            prof[name] = {"profiled_wall_ms": round(wall, 1), "device_ms": round(gpu, 1),
                          "host_gap_ms": round(max(0.0, wall - gpu), 1)}
            with open(os.path.join(a.profile, "%s.txt" % name.replace("+", "_")), "w") as fh:
                fh.write(p.key_averages().table(sort_by="self_device_time_total", row_limit=25))
    same = {n: hyps[n] == hyps[configs[0]] for n in configs if n not in ("beam_search", "graph")}
    if "graph" in configs and "beam_search" in configs:
        same["graph_vs_beam_search"] = hyps["graph"] == hyps["beam_search"]
    res = {"card": card(), "shape": a.shape, "layers": a.layers, "batch_size_val": a.batch_size_val, "cap": a.cap,
           "batches": a.batches, "ms_per_batch": {n: [round(x, 1) for x in v] for n, v in times.items()},
           "peak_gib": {n: round(v, 2) for n, v in peaks.items()}, "same_captions_as_first": same, "profile": prof}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "a") as fh:
            fh.write(line + "\n")
    if torch.distributed.is_initialized():
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
