"""Time every GEMM of the FT-Align cross encoder, the 1536-row text / visual GEMMs and the small-K weight gradients,
through ops.gemm.

Each row is one GEMM as ops.py issues it (attn_block_fwd / attn_block_bwd / ffn_block_fwd / ffn_block_bwd): its
operand majors, epilogue, bias, aux_in / aux_out and automatic tile-width / split-K plan.  The FT-Align cross encoder
runs T = 98304 rows (32 x 32 all-pairs sequences of 96 tokens); its self-attention takes the fused QKV-projection +
attention kernel, so the only QKV GEMMs of a cross layer are in the backward.  The text and visual stacks run 1536
rows (batch 32 x 48 tokens); the first-token cross layer's query, output and FFN weights see 1024 rows (one per
pair).  `--rows text` runs these small-K rows.

Prints one JSON line per GEMM: ms (CUDA events over enough launches for >= --min_s seconds, after a warm-up),
TFLOP/s (2 M N K), and the hardware bound max(FLOPs / 989 TFLOP/s, HBM bytes / 3.35 TB/s) — the H100 SXM data sheet's
dense bf16 rate and HBM3 bandwidth (700 W figures) — naming which of the two it is and the share of it reached.  HBM
bytes are the least the GEMM must move: A and B read once, the output written once (read and written for the
accumulating epilogue), aux_in read, aux_out written.  The card's name,
power limit and maximum SM clock are printed first, and the SM clock is read again after every row.

usage: python scripts/bench_gemm.py [--min_s 0.5] [--rows cross|text|all]
"""
import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from univl_b200 import ops  # noqa: E402

PEAK_FLOPS = 989e12
PEAK_BYTES = 3.35e12
H, I = 768, 3072
T_CROSS, T_TEXT, T_PAIRS = 98304, 1536, 1024
EPI_NAME = {ops.EPI_BIAS: "bias", ops.EPI_GELU: "bias_gelu", ops.EPI_GELU_BWD: "gelu_bwd", ops.EPI_ADD: "add",
            ops.EPI_F32: "bias_f32", ops.EPI_ATOMIC: "atomic_f32"}

# name: (T, kind, out features, in features, epilogue, bias)
#   fwd    Y[T, out]  = X[T, in] W[out, in]^T            (linear_fwd)
#   dgrad  dX[T, in]  = dY[T, out] W[out, in]            (linear_dgrad: W MN-major)
#   wgrad  dW[out, in] += dY[T, out]^T X[T, in]          (linear_wgrad: both MN-major, split-K, fp32)
CROSS = {
    "cross_attn_out_fwd": (T_CROSS, "fwd", H, H, ops.EPI_BIAS, True),
    "cross_ffn1_fwd_gelu": (T_CROSS, "fwd", I, H, ops.EPI_GELU, True),
    "cross_ffn2_fwd": (T_CROSS, "fwd", H, I, ops.EPI_BIAS, True),
    "cross_ffn2_wgrad": (T_CROSS, "wgrad", H, I, ops.EPI_ATOMIC, False),
    "cross_ffn2_dgrad_gelu_bwd": (T_CROSS, "dgrad", H, I, ops.EPI_GELU_BWD, False),
    "cross_ffn1_wgrad": (T_CROSS, "wgrad", I, H, ops.EPI_ATOMIC, False),
    "cross_ffn1_dgrad": (T_CROSS, "dgrad", I, H, ops.EPI_BIAS, False),
    "cross_attn_out_wgrad": (T_CROSS, "wgrad", H, H, ops.EPI_ATOMIC, False),
    "cross_attn_out_dgrad": (T_CROSS, "dgrad", H, H, ops.EPI_BIAS, False),
    "cross_qkv_wgrad": (T_CROSS, "wgrad", 3 * H, H, ops.EPI_ATOMIC, False),
    "cross_qkv_dgrad_add": (T_CROSS, "dgrad", 3 * H, H, ops.EPI_ADD, False),
    # the first-token cross layer (layer 2) projects K / V of all T rows (its queries are one row per pair)
    "cross2_kv_fwd": (T_CROSS, "fwd", 2 * H, H, ops.EPI_BIAS, True),
    "cross2_kv_dgrad": (T_CROSS, "dgrad", 2 * H, H, ops.EPI_BIAS, False),
    "cross2_kv_wgrad": (T_CROSS, "wgrad", 2 * H, H, ops.EPI_ATOMIC, False),
}
TEXT = {
    "text_qkv_fwd": (T_TEXT, "fwd", 3 * H, H, ops.EPI_BIAS, True),
    "text_attn_out_fwd": (T_TEXT, "fwd", H, H, ops.EPI_BIAS, True),
    "text_ffn1_fwd_gelu": (T_TEXT, "fwd", I, H, ops.EPI_GELU, True),
    "text_ffn2_fwd": (T_TEXT, "fwd", H, I, ops.EPI_BIAS, True),
    "text_ffn2_dgrad_gelu_bwd": (T_TEXT, "dgrad", H, I, ops.EPI_GELU_BWD, False),
    "text_qkv_dgrad_add": (T_TEXT, "dgrad", 3 * H, H, ops.EPI_ADD, False),
    "text_ffn2_wgrad": (T_TEXT, "wgrad", H, I, ops.EPI_ATOMIC, False),
    "text_ffn1_wgrad": (T_TEXT, "wgrad", I, H, ops.EPI_ATOMIC, False),
    "text_attn_out_wgrad": (T_TEXT, "wgrad", H, H, ops.EPI_ATOMIC, False),
    "text_qkv_wgrad": (T_TEXT, "wgrad", 3 * H, H, ops.EPI_ATOMIC, False),
    "visual_in_fwd": (T_TEXT, "fwd", H, 1024, ops.EPI_BIAS, True),
    "visual_in_wgrad": (T_TEXT, "wgrad", H, 1024, ops.EPI_ATOMIC, False),
    # the first-token cross layer's query, output and FFN weights see one row per pair (32 x 32)
    "cross2_q_wgrad": (T_PAIRS, "wgrad", H, H, ops.EPI_ATOMIC, False),
    "cross2_attn_out_wgrad": (T_PAIRS, "wgrad", H, H, ops.EPI_ATOMIC, False),
    "cross2_ffn1_wgrad": (T_PAIRS, "wgrad", I, H, ops.EPI_ATOMIC, False),
    "cross2_ffn2_wgrad": (T_PAIRS, "wgrad", H, I, ops.EPI_ATOMIC, False),
}


def nvsmi(query):
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=" + query, "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else None
    except (OSError, subprocess.SubprocessError):
        return None


def problem(T, kind, n_out, n_in, epi, has_bias, g):
    """(thunk launching the GEMM, M, N, K, HBM bytes)"""
    dev = "cuda"

    def rnd(*shape):
        return (torch.randn(*shape, device=dev, generator=g) * 0.5).to(torch.bfloat16)

    if kind == "fwd":
        a, b, M, N, K, a_mn, b_mn = rnd(T, n_in), rnd(n_out, n_in) * 0.1, T, n_out, n_in, 0, 0
    elif kind == "dgrad":
        a, b, M, N, K, a_mn, b_mn = rnd(T, n_out), rnd(n_out, n_in) * 0.1, T, n_in, n_out, 0, 1
    else:
        a, b, M, N, K, a_mn, b_mn = rnd(T, n_out), rnd(T, n_in), n_out, n_in, T, 1, 1
    f32 = epi in (ops.EPI_F32, ops.EPI_ATOMIC)
    out = (torch.zeros if f32 else torch.empty)(M, N, device=dev, dtype=torch.float32 if f32 else torch.bfloat16)
    bias = torch.randn(N, device=dev, generator=g) * 0.1 if has_bias else None
    aux_in = rnd(M, N) if epi in (ops.EPI_GELU_BWD, ops.EPI_ADD) else None
    aux_out = torch.empty(M, N, device=dev, dtype=torch.bfloat16) if epi == ops.EPI_GELU else None
    nbytes = 2 * (M * K + N * K) + out.element_size() * M * N * (2 if epi == ops.EPI_ATOMIC else 1)
    nbytes += 2 * M * N * ((aux_in is not None) + (aux_out is not None)) + (4 * N if has_bias else 0)

    def run():
        ops.gemm(a, b, M, N, K, out, epi=epi, bias=bias, aux_in=aux_in, aux_out=aux_out, a_mn=a_mn, b_mn=b_mn)
    return run, M, N, K, nbytes


def time_ms(fn, min_s, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(3):
        fn()
    e.record()
    torch.cuda.synchronize()
    iters = max(10, math.ceil(min_s * 1e3 / (s.elapsed_time(e) / 3)))
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters, iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min_s", type=float, default=0.5, help="seconds of launches timed per row")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rows", default="all", choices=["cross", "text", "all"])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gemm.py needs a CUDA device")
    print(json.dumps({"card": torch.cuda.get_device_name(0),
                      "power_limit_and_max_sm_clock": nvsmi("power.limit,clocks.max.sm")}), flush=True)
    rows = {**(CROSS if a.rows != "text" else {}), **(TEXT if a.rows != "cross" else {})}
    for i, (name, (T, kind, n_out, n_in, epi, has_bias)) in enumerate(rows.items()):
        g = torch.Generator(device="cuda").manual_seed(1000 + i)
        run, M, N, K, nbytes = problem(T, kind, n_out, n_in, epi, has_bias, g)
        ms, iters = time_ms(run, a.min_s, a.warmup)
        sm_clock = nvsmi("clocks.sm")
        flops = 2.0 * M * N * K
        t_flop, t_byte = flops / PEAK_FLOPS * 1e3, nbytes / PEAK_BYTES * 1e3
        bound_ms = max(t_flop, t_byte)
        print(json.dumps({"gemm": name, "M": M, "N": N, "K": K, "epilogue": EPI_NAME[epi], "ms": round(ms, 4),
                          "tflops": round(flops / ms * 1e-9, 1), "bound_ms": round(bound_ms, 4),
                          "bound": "compute" if t_flop >= t_byte else "hbm",
                          "share_of_bound": round(bound_ms / ms, 3), "launches": iters, "sm_clock": sm_clock}),
              flush=True)
        del run
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
