#!/usr/bin/env python
"""Benchmark of the UniVL data-parallel training hot path on H100 (BASELINE.json metric: video-text samples/sec).

    python bench.py --gpus N --steps K --warmup W            # this repo's CUDA path (N>1: launched under torchrun)
    python bench.py --impl reference --gpus N --steps K ...  # the reference algorithm on the host CPU cores

A "step" is one full training step of the hot path on one synthetic batch: zero-grad, UniVL.forward (loss), backward,
gradient all-reduce (N > 1), gradient clipping + BertAdam update.  Default workload = BASELINE.json configs[1]:
retrieval fine-tune, 12L text / 6L visual / 2L cross (FT-Align: `train_sim_after_cross`, B x B text-video pairs
through the cross encoder), per-GPU batch 32, max_words = max_frames = 48, bf16 tensor-core math with fp32 master
weights, dropout 0.1 active, random-init weights, synthetic (token-id, 1024-d S3D feature) batches.

One JSON line on stdout (rank 0).  `value` = whole-job samples/s with inputs resident in HBM; `e2e` = the same step
driven from pinned HOST buffers (H2D of every input and D2H of the loss inside the timed region); `roofline` = the
wgmma GEMM kernel's achieved TFLOP/s (CUDA events around its launches) against the bf16 peak;
`cpu_baseline` = the CPU oracle (port of the reference algorithm) timed on this box's host cores on a bounded sample.

`--dump-outputs DIR` (rank 0) writes what the last timed step computed as .npy files: `loss.npy`, and a fixed, seeded
sample of the updated fp32 master weights (`params_sample.npy`) and of rank 0's fp32 gradients from that step's backward
(`grads_sample.npy`; with one GPU these are the gradients the optimizer applied, with N > 1 the rank's local gradients
before the all-reduce), with `sample_index.npy` (float64) giving the positions in the flat parameter vector.  Inputs,
weights and dropout streams are seeded, so two builds run with the same arguments can be compared output for output.

N > 1: the gradients travel as a bf16 payload that the optimizer reads directly; for more than 2 GPUs the backward is cut at
text layer 6 (`--overlap_cuts`) so the all-reduce of the finished 61 % of the bytes runs under the rest of the backward
(univl_b200.ddp.PhasedBackward); `step_breakdown_ms` = rank 0's device time per segment of such a step.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


# Cutting the backward at text layer 6 lets the all-reduce of the finished 61 % of the gradient bytes run under the
# remaining backward; with two GPUs the collective slows the backward by what it hides, so the cut is only taken for
# world > 2.
AUTO_CUTS = "6"


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--mode", default="ft_align", choices=["ft_align", "ft_joint", "caption", "pretrain2"])
    ap.add_argument("--batch", type=int, default=32, help="per-GPU batch (weak scaling)")
    ap.add_argument("--max_words", type=int, default=48)
    ap.add_argument("--max_frames", type=int, default=48)
    ap.add_argument("--dropout", type=float, default=0.1)
    ap.add_argument("--cpu_sample_batch", type=int, default=8)
    ap.add_argument("--ref_kind", default="auto", choices=["auto", "reference", "port"],
                    help="--impl reference: the unmodified reference from oracle/_ref (auto: when staged) or the oracle port")
    ap.add_argument("--no_cpu_baseline", action="store_true")
    ap.add_argument("--no_e2e", action="store_true")
    ap.add_argument("--profile_steps", type=int, default=2)
    ap.add_argument("--grad_payload", default="bf16", choices=["bf16", "f32"],
                    help="N > 1: dtype of the gradient all-reduce payload (bf16 halves the NVLink bytes)")
    ap.add_argument("--overlap_cuts", default="auto", help="N > 1: text-encoder layers at which the backward is cut into "
                    "phases whose gradient all-reduce overlaps the next phase (univl_b200.ddp.PhasedBackward), e.g. "
                    "'9,5'; '' or 'off' = one all-reduce after the whole backward; auto = '6' for more than 2 GPUs, else off")
    ap.add_argument("--overlap_sms", type=int, default=0, help="SMs left to the overlapped all-reduce: NCCL_MAX_CTAS and "
                    "the reservation the persistent kernels of the overlapped phases size their grids for")
    ap.add_argument("--graph", type=int, default=1, help="1: replay the step as one CUDA graph (falls back to eager "
                    "launches if capture fails), 0: eager")
    ap.add_argument("--dump-outputs", dest="dump_outputs", default=None, metavar="DIR",
                    help="write the loss and a seeded sample of the updated weights and gradients of the last timed "
                    "step to DIR/<name>.npy (float32)")
    return ap.parse_args()


def workload_name(a):
    return "retrieval fine-tune %s, 12L text/6L visual%s, per-GPU batch %d, max_words=%d max_frames=%d" % (
        {"ft_align": "FT-Align (train_sim_after_cross, BxB pairs through 2L cross)", "ft_joint": "FT-Joint",
         "caption": "caption stage-two (+2L cross +3L decoder)", "pretrain2": "pretrain stage-two (5 objectives)"}[
            a.mode], "" if a.mode == "ft_joint" else "/2L cross", a.batch, a.max_words, a.max_frames)


def peaks():
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(path):
        with open(path) as fh:
            d = json.load(fh)
        return float(d.get("bf16_tflops_sustained", d.get("bf16_tflops", 1400.0))), "measured (MEASURED_PEAKS.json, sustained)"
    return 989.0, "H100 SXM data sheet, dense bf16 at 700 W (not reached by any measured kernel)"


class ClockSampler(threading.Thread):
    """nvidia-smi clocks / throttle reasons DURING the timed region"""

    def __init__(self, index):
        super().__init__(daemon=True)
        self.index, self.rows, self.stop_flag = index, [], False

    def run(self):
        q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
             "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
             "clocks_event_reasons.sw_power_cap")
        while not self.stop_flag:
            try:
                out = subprocess.run(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + q,
                                      "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=5)
                if out.returncode == 0 and out.stdout.strip():
                    self.rows.append([c.strip() for c in out.stdout.strip().split(",")])
            except Exception:
                pass
            time.sleep(0.1)

    def summary(self):
        sm = sorted(int(float(r[0])) for r in self.rows if r[0].replace(".", "").isdigit())
        if not sm:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["unavailable"]}
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = [n for i, n in enumerate(names) if any(len(r) > 3 + i and r[3 + i].lower().startswith("active")
                                                         for r in self.rows)]
        return {"sm_mhz": sm[len(sm) // 2], "sm_max_mhz": int(float(self.rows[0][1])), "reasons": reasons,
                "samples": len(sm)}


# ---------------------------------------------------------------------------------------------------------
def _host_threads(cap=32):
    """threads for the CPU arm: the cores this process may actually run on (cgroup / affinity aware), capped — the
    b=8 oracle sample's matrices are small (a few hundred rows) and 128 threads on a shared box thrash (measured: 240 s
    for a step that takes 8 s on 16 threads); the full-batch reference arm uses up to 64."""
    try:
        n = len(os.sched_getaffinity(0))
    except (AttributeError, OSError):
        n = os.cpu_count() or 1
    return max(1, min(n, cap))


class CpuReference:
    """The CPU oracle (the port of the reference algorithm; the Python reference itself cannot travel to the GPU box)
    on a bounded sample of the same workload: `cpu_sample_batch` videos/captions, i.e. b*b pair sequences through the
    cross encoder for FT-Align.  One step = forward + backward of that sample (fp32, all parameters' gradients)."""

    def __init__(self, a, threads=None):
        import torch
        from oracle import synth
        self.cores = threads or _host_threads()
        torch.set_num_threads(self.cores)
        self.b = a.cpu_sample_batch
        self.cfg = synth.task_config(mode=a.mode, batch_size=self.b, max_words=a.max_words, max_frames=a.max_frames)
        self.batch = synth.make_batch(self.cfg, seed=1234)
        self.sd = synth.make_state_dict(self.cfg, seed=0, weight_std=0.02)
        self.desc = "fwd+bwd steps of the CPU oracle at batch %d (%s), fp32, %d threads" % (
            self.b, "%d pair sequences" % (self.b * self.b) if a.mode == "ft_align" else "same layers", self.cores)

    def step(self):
        from tests.oracle_util import run_oracle
        t0 = time.time()
        run_oracle(self.cfg, self.batch, sd=self.sd, backward=True)
        return time.time() - t0


def cpu_reference_sample(a, threads=None):
    """the default run's `cpu_baseline` leg: 1 warm-up + up to 5 timed steps (bounded at ~30 s)
    -> (samples_per_s, seconds_per_step, cores, description)"""
    ref = CpuReference(a, threads)
    ref.step()  # warm-up (allocator, thread pool)
    times, t0 = [], time.time()
    while len(times) < 5 and (not times or time.time() - t0 < 30.0):
        times.append(ref.step())
    dt = sum(times) / len(times)
    return ref.b / dt, dt, ref.cores, "mean of %d " % len(times) + ref.desc


class RealReference:
    """The UNMODIFIED reference (microsoft/UniVL `modules.modeling.UniVL`, its own BertAdam) from oracle/_ref — staged
    by oracle/build_ref.py — on the host cores at the SAME per-rank batch as the GPU arm (BASELINE.md §3): torch CPU
    fp32, train mode with the config's dropout, random init (torch.manual_seed(0)), one step = zero_grad, forward,
    backward, clip_grad_norm_(1.0), BertAdam.step — the loop body of main_task_retrieval.py:333-353 without DDP."""

    def __init__(self, a, root):
        import types
        import torch
        from oracle import synth
        from tests.model_util import bert_dir
        for name in ("boto3", "botocore", "botocore.exceptions"):   # imported at modules/file_utils.py:20-21, unused
            if name not in sys.modules:
                sys.modules[name] = types.ModuleType(name)
        sys.modules["botocore.exceptions"].ClientError = type("ClientError", (Exception,), {})
        sys.modules["botocore"].exceptions = sys.modules["botocore.exceptions"]
        sys.path.insert(0, root)
        from modules.modeling import UniVL
        from modules.optimization import BertAdam
        self.torch = torch
        self.cores = _host_threads(cap=64)
        torch.set_num_threads(self.cores)
        self.b = a.batch
        cfg = synth.task_config(mode=a.mode, batch_size=a.batch, max_words=a.max_words, max_frames=a.max_frames)
        torch.manual_seed(0)
        self.model = UniVL.from_pretrained(bert_dir(), "visual-base", "cross-base", "decoder-base", task_config=cfg)
        for m in self.model.modules():
            if isinstance(m, torch.nn.Dropout):
                m.p = a.dropout
        self.model.train()
        named = list(self.model.named_parameters())
        no_decay = ["bias", "LayerNorm.bias", "LayerNorm.weight"]
        dec = [(n, p) for n, p in named if not any(nd in n for nd in no_decay)]
        nod = [(n, p) for n, p in named if any(nd in n for nd in no_decay)]
        lr, coef = 3e-5, 0.1
        groups = [{"params": [p for n, p in dec if "bert." in n], "weight_decay": 0.01, "lr": lr * coef},
                  {"params": [p for n, p in dec if "bert." not in n], "weight_decay": 0.01},
                  {"params": [p for n, p in nod if "bert." in n], "weight_decay": 0.0, "lr": lr * coef},
                  {"params": [p for n, p in nod if "bert." not in n], "weight_decay": 0.0}]
        self.opt = BertAdam(groups, lr=lr, warmup=0.1, schedule="warmup_linear", t_total=100000, weight_decay=0.01,
                            max_grad_norm=1.0)
        self.batch = synth.make_batch(cfg, seed=1234, b=a.batch)
        self.kind = "reference"
        self.desc = ("full training steps (fwd+bwd+clip+BertAdam) of the unmodified reference (oracle/_ref) at per-rank "
                     "batch %d, torch CPU fp32, dropout %.2f, %d threads" % (a.batch, a.dropout, self.cores))

    def step(self):
        t0 = time.time()
        self.opt.zero_grad()
        loss = self.model(**self.batch)
        loss.backward()
        self.torch.nn.utils.clip_grad_norm_(self.model.parameters(), 1.0)
        self.opt.step()
        return time.time() - t0


def run_reference_arm(a, budget_s=270.0):
    """`--impl reference`: W warm-up + K timed steps of the reference's own CPU path (rank 0 only) — the real reference
    from oracle/_ref when staged (kind "reference"), else the oracle port on a bounded sample (kind "port").  The run
    stops early once `budget_s` has passed (at least one timed step) so the driver's launch ends within minutes."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    from oracle import build_ref
    root = build_ref.ref_root() if a.ref_kind != "port" else None
    if a.ref_kind == "reference" and root is None:
        raise SystemExit("bench.py: --ref_kind reference but the reference is not staged (python oracle/build_ref.py)")
    t_start = time.time()
    if root is not None:
        ref = RealReference(a, root)
    else:
        ref = CpuReference(a)
        ref.kind = "port"
    n_warm = 0
    for _ in range(a.warmup):
        ref.step()
        n_warm += 1
        if time.time() - t_start > budget_s / 4:
            break
    times = []
    for _ in range(max(1, a.steps)):
        times.append(ref.step())
        if time.time() - t_start > budget_s:
            break
    dt = sum(times) / len(times)
    sps = ref.b / dt
    line = {"impl": "reference", "metric": "video-text samples/sec", "value": sps, "unit": "samples/s",
            "n_gpus": a.gpus, "steps": len(times), "warmup": n_warm, "ms_per_step": dt * 1e3,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": {"workload": workload_name(a) if ref.kind == "reference" else
                       workload_name(a).replace("per-GPU batch %d" % a.batch, "batch %d sample" % ref.b),
                       "note": "CPU: host cores only, no GPU; " + ref.desc},
            "cpu_baseline": {"value": sps, "unit": "samples/s", "cores": ref.cores, "kind": ref.kind,
                             "sample": ref.desc},
            "e2e": {"value": sps, "unit": "samples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line), flush=True)


# ---------------------------------------------------------------------------------------------------------
DUMP_SAMPLE = 1 << 21   # elements of the weight / gradient samples: 2 x 8 MB of float32 plus a 16 MB index


def dump_outputs(out_dir, loss, flat_params, flat_grads):
    """the last timed step's loss and a fixed, seeded sample of the flat fp32 weights and gradients -> out_dir/*.npy"""
    import numpy as np
    import torch
    os.makedirs(out_dir, exist_ok=True)
    n = flat_params.numel()
    g = torch.Generator().manual_seed(20240)
    idx = torch.randint(0, n, (DUMP_SAMPLE,), generator=g).sort().values
    idx_dev = idx.to(flat_params.device)
    arrays = {"loss": loss.detach().float().reshape(1).cpu(),
              "params_sample": flat_params.index_select(0, idx_dev).float().cpu(),
              "grads_sample": flat_grads.index_select(0, idx_dev).float().cpu(),
              "sample_index": idx.double()}
    for name, t in arrays.items():
        np.save(os.path.join(out_dir, name + ".npy"), t.numpy())


def main():
    a = parse()
    if a.impl == "reference":
        return run_reference_arm(a)

    import torch
    import torch.distributed as dist
    from oracle import synth
    from univl_b200 import ops, runtime as rt
    from univl_b200.ddp import FlatGradReducer, PhasedBackward
    from univl_b200.optim import FusedBertAdam
    from tests.model_util import bert_dir

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device — the product path has no CPU fallback")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    cuts = a.overlap_cuts
    if cuts == "auto":
        cuts = AUTO_CUTS if world > 2 else "off"
    overlap = world > 1 and a.graph and cuts not in ("", "off", "0")
    if world > 1:
        if overlap and a.overlap_sms > 0:
            # the all-reduce that runs under the next backward phase gets a fixed SM allowance; the phase's persistent
            # kernels are launched on the remaining SMs (univl_set_reserved_sms) instead of queueing a second wave
            os.environ.setdefault("NCCL_MAX_CTAS", str(a.overlap_sms))
        dist.init_process_group("nccl", device_id=dev)

    from univl_b200.modules.modeling import UniVL
    cfg = synth.task_config(mode=a.mode, batch_size=a.batch * world, n_gpu=world, max_words=a.max_words,
                            max_frames=a.max_frames)
    torch.manual_seed(0)
    model = UniVL.from_pretrained(bert_dir(), "visual-base", "cross-base", "decoder-base", task_config=cfg)
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = a.dropout
    model.to(dev).train()

    # optimizer param groups exactly as the reference driver builds them (main_task_retrieval.py:173-190)
    named = list(model.named_parameters())
    no_decay = ["bias", "LayerNorm.bias", "LayerNorm.weight"]
    dec = [(n, p) for n, p in named if not any(nd in n for nd in no_decay)]
    nod = [(n, p) for n, p in named if any(nd in n for nd in no_decay)]
    lr, coef = 3e-5, 0.1
    groups = [{"params": [p for n, p in dec if "bert." in n], "weight_decay": 0.01, "lr": lr * coef},
              {"params": [p for n, p in dec if "bert." not in n], "weight_decay": 0.01},
              {"params": [p for n, p in nod if "bert." in n], "weight_decay": 0.0, "lr": lr * coef},
              {"params": [p for n, p in nod if "bert." not in n], "weight_decay": 0.0}]
    opt = FusedBertAdam(groups, lr=lr, warmup=0.1, t_total=100000, max_grad_norm=1.0, global_clip_norm=1.0,
                        grad_scale=1.0 / world, model=model)
    opt._build()
    reducer = FlatGradReducer(opt.p, opt.g, n_buckets=4, compress="bf16" if a.grad_payload == "bf16" else None)
    phased = None
    if overlap:
        n_text = len(model.bert.encoder.layer)
        cut_layers = [int(c) for c in cuts.split(",") if 0 < int(c) < n_text]
        if cut_layers:
            phased = PhasedBackward(model, opt.flat, cut_layers)

    host_batch = synth.make_batch(cfg, seed=1234 + rank, b=a.batch)
    host_batch = {k: v.pin_memory() for k, v in host_batch.items()}
    dev_batch = {k: v.to(dev) for k, v in host_batch.items()}
    h2d_bytes = sum(v.numel() * v.element_size() for v in host_batch.values())

    def fwd_bwd(batch):
        opt.zero_grad()
        if phased is not None:
            phased.begin()
        loss = model(**batch)
        if phased is not None:
            phased.backward(0, loss)
            for ph in range(1, phased.n_phases):
                phased.backward(ph)
        else:
            loss.backward()
        return loss

    def step(batch):
        loss = fwd_bwd(batch)
        reducer.all_reduce()
        opt.step()
        return loss

    def stage(msg):
        if os.environ.get("UNIVL_BENCH_VERBOSE"):
            sys.stderr.write("[bench rank %d] %s\n" % (rank, msg))
            sys.stderr.flush()

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    stage("model + optimizer built; warm-up")
    for _ in range(a.warmup):
        step(dev_batch)
    barrier()
    stage("warm-up done")

    # ---- optional: capture the whole step (zero-grad, fwd, bwd, all-reduce, optimizer) into one CUDA graph.  Inputs
    # live in static device buffers; dropout masks still change every replay (device-side RNG epoch). ----
    eager_step = step
    launches_per_step = None
    graphed = False
    if a.graph:
        try:
            n0 = rt.launch_count()
            static_batch = {k: v.clone() for k, v in dev_batch.items()}
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                eager_step(static_batch)
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            n0 = rt.launch_count()
            # N > 1: the NCCL all-reduce stays an eager call between graphs.  Without phases: forward+backward | all-reduce
            # | optimizer.  With phases: forward + backward phase 0 | async all-reduce of phase 0's finished gradient runs
            # || backward phase 1 | async all-reduce of phase 1's runs || ... | wait | optimizer -- the exchange of one
            # phase rides under the compute of the next (what DDP's bucket hooks do in the reference).
            graph = torch.cuda.CUDAGraph()
            graph_opt = None
            phase_graphs = []
            with torch.cuda.graph(graph):
                if world == 1:
                    static_loss = eager_step(static_batch)
                elif phased is None:
                    static_loss = fwd_bwd(static_batch)
                    reducer.pack()          # fp32 gradients -> bf16 payload, inside the backward graph
                else:
                    opt.zero_grad()
                    phased.begin()
                    static_loss = model(**static_batch)
                    phased.backward(0, static_loss)
                    reducer.pack(phased.ranges[0])
            if phased is not None:
                for ph in range(1, phased.n_phases):
                    g_ph = torch.cuda.CUDAGraph()
                    rt.reserve_sms(a.overlap_sms)   # this phase shares the GPU with an all-reduce
                    try:
                        with torch.cuda.graph(g_ph, pool=graph.pool()):
                            phased.backward(ph)
                            reducer.pack(phased.ranges[ph])
                    finally:
                        rt.reserve_sms(0)
                    phase_graphs.append(g_ph)
            if world > 1:
                graph_opt = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph_opt, pool=graph.pool()):
                    if reducer.compress is not None:
                        opt.grad_payload = reducer.payload   # the optimizer reads the summed bf16 payload directly
                    opt.step()
                    opt.grad_payload = None
            launches_per_step = rt.launch_count() - n0
            torch.cuda.synchronize()
            stage("graphs captured")

            def step(batch, marks=None):
                def mark(tag):
                    if marks is not None:
                        ev = torch.cuda.Event(enable_timing=True)
                        ev.record()
                        marks.append((tag, ev))
                if batch is not static_batch:
                    for k, v in batch.items():
                        static_batch[k].copy_(v, non_blocking=True)
                mark("start")
                graph.replay()
                if phased is not None:
                    mark("forward + backward phase 0")
                    works = reducer.all_reduce_ranges(phased.ranges[0])
                    for ph, g_ph in enumerate(phase_graphs, 1):
                        g_ph.replay()
                        mark("backward phase %d (under the all-reduce of phase %d)" % (ph, ph - 1))
                        works += reducer.all_reduce_ranges(phased.ranges[ph])
                    for w in works:
                        w.wait()
                    mark("exposed all-reduce")
                    graph_opt.replay()
                    mark("optimizer")
                elif graph_opt is not None:
                    mark("forward + backward")
                    reducer.all_reduce(packed=True)
                    mark("all-reduce")
                    graph_opt.replay()
                    mark("optimizer")
                return static_loss
            for _ in range(2):
                step(static_batch)
            barrier()
            graphed = True
            dev_batch = static_batch
        except Exception as exc:  # noqa: BLE001
            sys.stderr.write("bench.py: CUDA graph capture failed (%r); timing eager launches instead\n" % (exc,))
            step = eager_step
            torch.cuda.synchronize()

    sampler = ClockSampler(local) if rank == 0 else None
    if sampler:
        sampler.start()

    stage("timed region")
    # ---- timed region 1: inputs resident in HBM ----
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    launches0 = rt.launch_count()
    barrier()
    e0.record()
    for _ in range(a.steps):
        loss = step(dev_batch)
    e1.record()
    barrier()
    ms = e0.elapsed_time(e1) / a.steps
    launches = (launches_per_step * a.steps) if graphed else (rt.launch_count() - launches0)
    loss_val = float(loss.detach())
    if a.dump_outputs and rank == 0:
        dump_outputs(a.dump_outputs, loss, opt.p, opt.g)

    # where a multi-GPU step goes (rank 0's device clock, 5 extra steps outside the timed region)
    breakdown = None
    if world > 1 and graphed:
        acc = {}
        for _ in range(5):
            marks = []
            step(dev_batch, marks)
            torch.cuda.synchronize()
            for (_, e_a), (tag, e_b) in zip(marks[:-1], marks[1:]):
                acc[tag] = acc.get(tag, 0.0) + e_a.elapsed_time(e_b) / 5
        breakdown = acc
        barrier()

    # ---- timed region 2: end to end from pinned host buffers (H2D of inputs + D2H of the loss every step) ----
    e2e = None
    if not a.no_e2e:
        # The loss of every step is read back into pinned host memory by an asynchronous D2H copy on the step's stream
        # (what a training loop that logs the loss does); the host synchronises once, after the last step, so host-side
        # jitter queues behind the device instead of stalling it.
        # The inputs of step i+1 are prefetched while step i computes, as any input pipeline does: H2D from the pinned
        # host batch into one of two staging sets on a copy stream, then a device-to-device copy into the graph's static
        # input tensors at the head of the step.  Every step still moves all its input bytes host -> device and its loss
        # device -> host inside the timed region.
        loss_host = torch.zeros(a.steps + 2, dtype=torch.float32).pin_memory()
        copy_stream = torch.cuda.Stream()
        stage_sets = [{k: torch.empty_like(v) for k, v in dev_batch.items()} for _ in range(2)]
        staged = [torch.cuda.Event(), torch.cuda.Event()]      # H2D into set s finished
        consumed = [torch.cuda.Event(), torch.cuda.Event()]    # set s copied out by the compute stream
        for ev in consumed:
            ev.record(torch.cuda.current_stream())

        def prefetch(i):
            s_ = i % 2
            copy_stream.wait_event(consumed[s_])
            with torch.cuda.stream(copy_stream):
                for k, v in host_batch.items():
                    stage_sets[s_][k].copy_(v, non_blocking=True)
                staged[s_].record(copy_stream)

        def e2e_step(i, slot):
            s_ = i % 2
            cur = torch.cuda.current_stream()
            cur.wait_event(staged[s_])
            if graphed:
                for k, v in stage_sets[s_].items():
                    dev_batch[k].copy_(v, non_blocking=True)
                batch = dev_batch
            else:
                batch = {k: v.clone() for k, v in stage_sets[s_].items()}
            consumed[s_].record(cur)
            prefetch(i + 1)
            loss_host[slot:slot + 1].copy_(step(batch).detach().reshape(1), non_blocking=True)
        prefetch(0)
        for i in range(2):
            e2e_step(i, a.steps + i)
        barrier()
        e0.record()
        for i in range(a.steps):
            e2e_step(i + 2, i)
        e1.record()
        barrier()
        ms_e2e = e0.elapsed_time(e1) / a.steps
        loss_val = float(loss_host[a.steps - 1])
    if sampler:
        sampler.stop_flag = True
        sampler.join(timeout=3)

    # ---- roofline of the dominant kernel: CUDA events around every wgmma GEMM launch on the launching stream ----
    # univl_gemm_plan reports which kernel each call launches (today always 1, the persistent wgmma kernel).
    from univl_b200 import lib as _lib
    prof = {1: {"flops": 0.0, "events": []}}
    orig_gemm = ops.gemm

    def timed_gemm(a_, b_, M, N, K, out, *args, **kw):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        r = orig_gemm(a_, b_, M, N, K, out, *args, **kw)
        e.record()
        epi = kw.get("epi", args[0] if args else 0)
        v = prof[int(_lib.load().univl_gemm_plan(M, N, K, int(epi), int(kw.get("block_n", 0)),
                                                 int(kw.get("split_k", 0))))]
        v["events"].append((s, e))
        v["flops"] += 2.0 * M * N * K
        return r
    # the fused QKV-projection + attention kernel (north_star's headline kernel) and its backward, timed the same way
    fa = {"fwd": {"flops": 0.0, "events": []}, "bwd": {"flops": 0.0, "events": []}}
    orig_fa_fwd, orig_fa_bwd = ops.fused_qkv_attention_fwd, ops.fused_attention_bwd

    def timed_fa_fwd(x_, wqkv_, bqkv_, n_seq_, S_, *args, **kw):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        r = orig_fa_fwd(x_, wqkv_, bqkv_, n_seq_, S_, *args, **kw)
        e.record()
        T_, H_ = x_.shape
        fa["fwd"]["events"].append((s, e))
        fa["fwd"]["flops"] += 2.0 * T_ * 3 * H_ * H_ + 4.0 * T_ * S_ * H_       # projection + QK^T + PV
        return r

    def timed_fa_bwd(qkv_, o_, lse_, d_o_, dqkv_, n_seq_, S_, *args, **kw):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        r = orig_fa_bwd(qkv_, o_, lse_, d_o_, dqkv_, n_seq_, S_, *args, **kw)
        e.record()
        fa["bwd"]["events"].append((s, e))
        fa["bwd"]["flops"] += 10.0 * o_.shape[0] * S_ * o_.shape[1]               # S, dP, dQ, dK, dV products
        return r
    ops.gemm = timed_gemm
    ops.fused_qkv_attention_fwd, ops.fused_attention_bwd = timed_fa_fwd, timed_fa_bwd
    two_stream = os.environ.get("UNIVL_TWO_STREAM")
    os.environ["UNIVL_TWO_STREAM"] = "0"   # per-launch durations are only meaningful when kernels do not share the GPU
    if a.profile_steps > 0:
        eager_step(dev_batch)              # untimed: lets the caching allocator settle in this (single-stream) mode
    torch.cuda.synchronize()
    for v in list(prof.values()) + list(fa.values()):
        v["events"].clear()
        v["flops"] = 0.0
    for _ in range(a.profile_steps):
        eager_step(dev_batch)
    torch.cuda.synchronize()
    if two_stream is None:
        del os.environ["UNIVL_TWO_STREAM"]
    else:
        os.environ["UNIVL_TWO_STREAM"] = two_stream
    ops.gemm = orig_gemm
    ops.fused_qkv_attention_fwd, ops.fused_attention_bwd = orig_fa_fwd, orig_fa_bwd
    fa_out = {}
    for k, v in fa.items():
        ms_k = sum(s.elapsed_time(e) for s, e in v["events"])
        big = max((s.elapsed_time(e) for s, e in v["events"]), default=0.0)
        fa_out[k] = {"ms_per_step": ms_k / max(1, a.profile_steps), "launches_per_step": len(v["events"]) / max(1, a.profile_steps),
                     "tflops": v["flops"] / (ms_k * 1e-3) / 1e12 if ms_k > 0 else 0.0, "largest_launch_ms": big}
    per = {}
    for k, v in prof.items():
        ms_k = sum(s.elapsed_time(e) for s, e in v["events"])
        per[k] = {"ms": ms_k, "n": len(v["events"]), "flops": v["flops"],
                  "tflops": v["flops"] / (ms_k * 1e-3) / 1e12 if ms_k > 0 else 0.0}
    dom = per[1]
    gemm_ms, n_gemm, achieved = dom["ms"], dom["n"], dom["tflops"]
    peak, peak_src = peaks()

    # max over ranks
    t = torch.tensor([ms, ms_e2e if not a.no_e2e else 0.0], device=dev, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms, ms_e2e_max = float(t[0]), float(t[1])
    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return

    samples = a.batch * world
    line = {
        "metric": "video-text samples/sec", "value": samples / (ms * 1e-3), "unit": "samples/s", "n_gpus": world,
        "steps": a.steps, "warmup": a.warmup, "ms_per_step": ms, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
        "config": {"workload": workload_name(a), "global_batch": samples, "parallelism": "dp%d" % world,
                   "dropout": a.dropout, "optimizer": "fused BertAdam + clip (in timed region)",
                   "grad_allreduce": "none" if world == 1 else ("NCCL sum, %s payload, %s" % (
                       a.grad_payload, "after backward" if phased is None or not graphed else
                       "overlapped with backward: %d phases cut at text layers %s" % (phased.n_phases, phased.cuts))),
                   "launch": "cuda-graph replay" if graphed else "eager",
                   "l2": "per-step working set (~6 GB of activations at FT-Align b=32) exceeds the 50 MB L2"},
        "gpu_launches": launches, "loss": loss_val,
        **({"step_breakdown_ms": breakdown} if breakdown else {}),
        "roofline": {"bound": "tensor", "achieved": achieved, "peak": peak, "unit": "TFLOP/s",
                     "frac": achieved / peak if peak else None,
                     "kernel": "gemm_wgmma_kernel",
                     "launches_per_step": n_gemm / max(1, a.profile_steps),
                     "gemm_ms_per_step": gemm_ms / max(1, a.profile_steps), "peak_source": peak_src,
                     "algorithmic_flops_per_step": dom["flops"] / max(1, a.profile_steps)},
        "clocks": sampler.summary() if sampler else None,
        "fused_attention": fa_out,
    }
    if not a.no_e2e:
        line["e2e"] = {"value": samples / (ms_e2e_max * 1e-3), "unit": "samples/s", "h2d_bytes_per_step": h2d_bytes,
                       "d2h_bytes_per_step": 4, "ms_per_step": ms_e2e_max}
    if world > 1:
        dist.destroy_process_group()
    if not a.no_cpu_baseline and world == 1:
        sps, dt, cores, desc = cpu_reference_sample(a)
        line["cpu_baseline"] = {"value": sps, "unit": "samples/s", "cores": cores, "kind": "port", "sample": desc,
                                "seconds": dt}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
