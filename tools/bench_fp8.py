"""python tools/bench_fp8.py [--out DIR] : bf16 against the FP8 modes on the bench's networks (SUPIR-v0 + SDXL-base shapes, random
weights), in one process. Modes: the FP8 linears (ControlWrapper.dtype = torch.float8_e4m3fn), + convs (.fp8_convs = True),
+ attention (.fp8_attention = True), + convs + attention.

  1. one denoiser call of the bench plan (34 rows = 17 windows x CFG pair of 128^2 latent), the modes alternated 3x each (--windows), CUDA
     events around 5 graph replays per window, with the card, its power limit and the median SM clock of each window; the same
     for one untiled CFG-pair call of a 256^2 latent (2 rows, the shape of the cfg2 workload);
  2. the per-launch shape table of one eager call in each mode and shape (the SUPIR_BENCH_DUMP_SHAPES form of bench.py),
     GEMM-class launches (gemm, gemm_fp8, conv3x3, conv3x3_fp8), the attentions (attention, attention_fp8 and its operand pass
     attention_quant_fp8), the quantization passes (layernorm_quant, quantize_rows) and the GroupNorm applies (groupnorm_apply,
     groupnorm_apply_quant) each timed with a CUDA-event pair;
  3. the cfg3 EDM step (49 windows, tile batch 17) in every mode, alternated, without the VAE (a random latent);
  4. the resident bytes of the packed networks in each mode.

Prints one JSON line and writes it (and the shape table) under --out. Reuses bench.engine_config / ClockSampler unchanged."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

FP8, BF = torch.float8_e4m3fn, torch.bfloat16
# (ControlWrapper.dtype, .fp8_convs, .fp8_attention)
MODES = {"bf16": (BF, False, False), "fp8": (FP8, False, False), "fp8_convs": (FP8, True, False), "fp8_attn": (FP8, False, True),
         "fp8_convs_attn": (FP8, True, True)}


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return {"nvidia_smi": q, "torch_name": torch.cuda.get_device_name(0)}


def packed_bytes(net):
    seen, n = set(), 0
    for m in (net.diffusion_model, net.control_model):
        for mod in m.modules():
            for k, v in vars(mod).items():
                if not k.startswith("_") or k == "_ln":
                    continue
                for t in (v if isinstance(v, tuple) else (v,)):
                    if torch.is_tensor(t) and t.is_cuda and id(t) not in seen:
                        seen.add(id(t))
                        n += t.numel() * t.element_size()
    return n


def set_mode(net, mode):
    net.dtype, net.fp8_convs, net.fp8_attention = MODES[mode]
    net.pack()
    torch.cuda.empty_cache()


def call_inputs(B, side):
    x = torch.randn(B, 4, side, side, device="cuda")
    cond = {"crossattn": torch.randn(B, 77, 2048, device="cuda"), "vector": torch.randn(B, 2816, device="cuda"),
            "control": torch.randn(B, 4, side, side, device="cuda")}
    return x, torch.full((B,), 500.0, device="cuda"), cond


def time_call(net, args, reps):
    clocks = bench.ClockSampler(0)
    clocks.start()
    for _ in range(2):
        net(*args, control_scale=1.0)
    torch.cuda.synchronize()
    clocks.mark()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        net(*args, control_scale=1.0)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps, clocks.stop()


def shape_table(net):
    """One eager run of the captured plan with a CUDA-event pair around every GEMM-class, quantization and GroupNorm-apply launch.
    Memory-bound rows report GB/s from the bytes per element they move (`gbs`)."""
    from supir_b200 import ops
    rec, orig = [], {}

    def wrap(name, flop):
        f = getattr(ops, name)
        orig[name] = f

        def g(*a, **kw):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = f(*a, **kw)
            e1.record()
            fl = flop(*a, **kw)
            rec.append((e0, e1, fl[0], fl[1], fl[2] if len(fl) > 2 else 0))
            return r
        setattr(ops, name, g)

    wrap("gemm", lambda a, w, out, **kw: (2.0 * a.shape[0] * w.shape[0] * a.shape[1], ("gemm", a.shape[0], w.shape[0], a.shape[1], kw.get("act", 0))))
    wrap("gemm_fp8", lambda aq, sa, wq, sw, out, **kw: (2.0 * aq.shape[0] * wq.shape[0] * aq.shape[1],
                                                       ("gemm_fp8", aq.shape[0], wq.shape[0], aq.shape[1], kw.get("act", 0))))
    wrap("conv3x3", lambda x, B, H, W, wp, out, **kw: (2.0 * x.shape[0] * wp.shape[0] * wp.shape[1], ("conv3x3", x.shape[0], wp.shape[0], wp.shape[1], kw.get("act", 0))))
    wrap("conv3x3_fp8", lambda xq, xs, B, H, W, wq, ws, out, **kw: (2.0 * xq.shape[0] * wq.shape[0] * wq.shape[1],
                                                                  ("conv3x3_fp8", xq.shape[0], wq.shape[0], wq.shape[1], kw.get("act", 0))))
    # bytes per element: bf16 read + e4m3 write (3), bf16 read + bf16 write (4), bf16 read twice + e4m3 write (5)
    wrap("quantize_rows", lambda x, q, s: (0.0, ("quantize_rows", x.shape[0], 0, x.shape[1], 0), 3))
    wrap("layernorm_quant", lambda x, g, b, q, s, eps=1e-5: (0.0, ("layernorm_quant", x.shape[0], 0, x.shape[1], 0), 3))
    wrap("groupnorm_apply", lambda x, B, HW, out, *a, **kw: (0.0, ("groupnorm_apply", x.shape[0], 0, x.shape[1], 0), 4))
    wrap("groupnorm_apply_quant", lambda x, B, HW, *a, **kw: (0.0, ("groupnorm_apply_quant", x.shape[0], 0, x.shape[1], 0), 5))
    # attentions: M = B * Lq, N = Lk, K = heads * 64, 4 M N K flop (Q K^T and P V); the operand pass as bf16 q, k, v read + k, v
    # read again by the amax pass + e4m3 written: 2 (Lq + 4 Lk) + Lq + 2 Lk bytes per (row, column) of M x K, taken as Lq = Lk
    wrap("attention", lambda q, k, v, out, B, heads, Lq, Lk, **kw: (4.0 * B * Lq * Lk * heads * 64, ("attention", B * Lq, Lk, heads * 64, 0)))
    wrap("attention_fp8", lambda q8, sq, k8, sk, vt8, sv, out, B, heads, Lq, Lk, **kw: (4.0 * B * Lq * Lk * heads * 64,
                                                                                        ("attention_fp8", B * Lq, Lk, heads * 64, 0)))
    wrap("attention_quant_fp8", lambda q, k, v, B, heads, Lq, Lk, *a, **kw: (0.0, ("attention_quant_fp8", B * Lq, Lk, heads * 64, 0), 13))
    plan = next(iter(net._plans.values()))
    try:
        plan._run()
        torch.cuda.synchronize()
    finally:
        for k, f in orig.items():
            setattr(ops, k, f)
    agg = {}
    for e0, e1, fl, key, bpe in rec:
        a = agg.setdefault(key, [0, 0.0, 0.0, bpe])
        a[0] += 1
        a[1] += e0.elapsed_time(e1)
        a[2] += fl
    rows = sorted(({"op": k[0], "M": k[1], "N": k[2], "K": k[3], "act": k[4], "count": v[0], "ms": round(v[1], 3),
                    "tflops": round(v[2] / (v[1] * 1e-3) / 1e12, 1) if v[2] else None,
                    "gbs": round(k[1] * k[3] * v[3] / (v[1] / v[0] * 1e-3) / 1e9, 1) if not v[2] else None}
                   for k, v in agg.items()), key=lambda r: -r["ms"])
    return {"total_ms": sum(r["ms"] for r in rows), "rows": rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=tempfile.gettempdir(), help="directory for bench_fp8.json (default: the temporary directory)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--windows", type=int, default=3, help="times every mode is timed, alternated with the others")
    args = ap.parse_args()
    torch.manual_seed(1234)
    res = {"card": card()}
    w = bench.WORKLOADS["cfg3"]
    m = bench.build_engine(w, "cuda:0", 1)
    net = m.model
    # ---- 1. one 34-row denoiser call of 128^2 latent (tiled cfg3), one 2-row call of 256^2 latent (untiled cfg2) ----
    res["resident_bytes"] = {}
    for key, (B, side) in (("call_34rows_128", (34, 128)), ("call_2rows_256", (2, 256))):
        call_args = call_inputs(B, side)
        calls = {mode: [] for mode in MODES}
        for rep in range(args.windows):
            for mode in MODES:
                set_mode(net, mode)
                res["resident_bytes"][mode] = packed_bytes(net)
                ms, clk = time_call(net, call_args, args.reps)
                calls[mode].append({"ms": ms, "sm_mhz": clk.get("sm_mhz"), "reasons": clk.get("reasons")})
                if rep == args.windows - 1:
                    res[f"{mode}_shape_table" + ("" if side == 128 else "_256")] = shape_table(net)
        res[key] = {k: {"median_ms": float(np.median([c["ms"] for c in v])), "windows": v} for k, v in calls.items()}
        del call_args
        net.clear_plans()
        torch.cuda.empty_cache()
    # ---- 3. the cfg3 EDM step (no VAE: a random latent) ----
    from supir_b200 import sampling
    latent = w["in_px"] * w["upscale"] // 8
    c = {"crossattn": torch.randn(1, 77, 2048, device="cuda"), "vector": torch.randn(1, 2816, device="cuda")}
    uc = {"crossattn": torch.randn(1, 77, 2048, device="cuda"), "vector": torch.randn(1, 2816, device="cuda")}
    z = 0.5 * torch.randn(1, 4, latent, latent, device="cuda")
    steps = {mode: [] for mode in MODES}
    for rep in range(args.windows):
        for mode in MODES:
            set_mode(net, mode)
            smp = m.make_sampler(w["steps"], -1.0, 5, 1.01, 4.0, True, 1.0)
            run = smp.begin(sampling.FusedDenoiser(m.denoiser, net), torch.randn_like(z), dict(c, control=z), dict(uc, control=z),
                            x_center=z, control_scale=1.0)
            run.step(0)
            torch.cuda.synchronize()
            clocks = bench.ClockSampler(0)
            clocks.start()
            run.step(1)
            torch.cuda.synchronize()
            clocks.mark()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(2, 2 + args.steps):
                run.step(i)
            e1.record()
            torch.cuda.synchronize()
            clk = clocks.stop()
            steps[mode].append({"ms": e0.elapsed_time(e1) / args.steps, "sm_mhz": clk.get("sm_mhz"), "reasons": clk.get("reasons"),
                                "finite": bool(torch.isfinite(run.x).all())})
            del run, smp
            net.clear_plans()
            torch.cuda.empty_cache()
    res["cfg3_step"] = {k: {"median_ms": float(np.median([s["ms"] for s in v])), "windows": v} for k, v in steps.items()}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "bench_fp8.json"), "w") as f:
        json.dump(res, f, indent=1)
    short = {k: v for k, v in res.items() if "shape_table" not in k}
    short["fp8_shape_table_top"] = res["fp8_shape_table"]["rows"][:12]
    short["fp8_convs_shape_table_top"] = res["fp8_convs_shape_table"]["rows"][:12]
    # the per-launch rows the convs option changes: 3x3 convolutions and GroupNorm applies, before (fp8) and after (fp8_convs)
    conv_ops = ("conv3x3", "conv3x3_fp8", "groupnorm_apply", "groupnorm_apply_quant")
    for mode in ("fp8", "fp8_convs"):
        t = res[f"{mode}_shape_table"]["rows"]
        short[f"{mode}_conv_rows"] = [r for r in t if r["op"] in conv_ops]
        short[f"{mode}_ms_by_op"] = {op: round(sum(r["ms"] for r in t if r["op"] == op), 3) for op in sorted({r["op"] for r in t})}
    # the per-launch rows the attention option changes, at both shapes and in every mode
    attn_ops = ("attention", "attention_fp8", "attention_quant_fp8")
    for mode in MODES:
        for suffix in ("", "_256"):
            t = res[f"{mode}_shape_table{suffix}"]["rows"]
            short[f"{mode}_attention_rows{suffix}"] = [r for r in t if r["op"] in attn_ops]
    print(json.dumps(short))


if __name__ == "__main__":
    main()
