"""python tools/bench_fp8.py [--out DIR] : bf16 against the FP8 linears mode (ControlWrapper.dtype = torch.float8_e4m3fn) on
the bench's networks (SUPIR-v0 + SDXL-base shapes, random weights), in one process:

  1. one denoiser call of the bench plan (34 rows = 17 windows x CFG pair of 128^2 latent), bf16 and FP8 alternated 3x each,
     CUDA events around 5 graph replays per window, with the card, its power limit and the median SM clock of each window;
  2. the per-launch shape table of one eager FP8 call (the SUPIR_BENCH_DUMP_SHAPES form of bench.py), GEMM-class launches and
     the quantization passes (layernorm_quant, quantize_rows) each timed with a CUDA-event pair;
  3. the cfg3 EDM step (49 windows, tile batch 17) in both modes, alternated, without the VAE (a random latent);
  4. the resident bytes of the packed networks in both modes.

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
MODES = {"bf16": BF, "fp8": FP8}


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
    net.dtype = MODES[mode]
    net.pack()
    torch.cuda.empty_cache()


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
    """One eager run of the captured plan with a CUDA-event pair around every GEMM-class and quantization launch."""
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
            rec.append((e0, e1) + flop(*a, **kw))
            return r
        setattr(ops, name, g)

    wrap("gemm", lambda a, w, out, **kw: (2.0 * a.shape[0] * w.shape[0] * a.shape[1], ("gemm", a.shape[0], w.shape[0], a.shape[1], kw.get("act", 0))))
    wrap("gemm_fp8", lambda aq, sa, wq, sw, out, **kw: (2.0 * aq.shape[0] * wq.shape[0] * aq.shape[1],
                                                       ("gemm_fp8", aq.shape[0], wq.shape[0], aq.shape[1], kw.get("act", 0))))
    wrap("conv3x3", lambda x, B, H, W, wp, out, **kw: (2.0 * x.shape[0] * wp.shape[0] * wp.shape[1], ("conv3x3", x.shape[0], wp.shape[0], wp.shape[1], kw.get("act", 0))))
    wrap("quantize_rows", lambda x, q, s: (0.0, ("quantize_rows", x.shape[0], 0, x.shape[1], 0)))
    wrap("layernorm_quant", lambda x, g, b, q, s, eps=1e-5: (0.0, ("layernorm_quant", x.shape[0], 0, x.shape[1], 0)))
    plan = next(iter(net._plans.values()))
    try:
        plan._run()
        torch.cuda.synchronize()
    finally:
        for k, f in orig.items():
            setattr(ops, k, f)
    agg = {}
    for e0, e1, fl, key in rec:
        a = agg.setdefault(key, [0, 0.0, 0.0])
        a[0] += 1
        a[1] += e0.elapsed_time(e1)
        a[2] += fl
    rows = sorted(({"op": k[0], "M": k[1], "N": k[2], "K": k[3], "act": k[4], "count": v[0], "ms": round(v[1], 3),
                    "tflops": round(v[2] / (v[1] * 1e-3) / 1e12, 1) if v[2] else None,
                    "gbs": round(k[1] * k[3] * 3 / (v[1] / v[0] * 1e-3) / 1e9, 1) if not v[2] else None}
                   for k, v in agg.items()), key=lambda r: -r["ms"])
    return {"total_ms": sum(r["ms"] for r in rows), "rows": rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=tempfile.gettempdir(), help="directory for bench_fp8.json (default: the temporary directory)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=2)
    args = ap.parse_args()
    torch.manual_seed(1234)
    res = {"card": card()}
    w = bench.WORKLOADS["cfg3"]
    m = bench.build_engine(w, "cuda:0", 1)
    net = m.model
    # ---- 1. one 34-row denoiser call of 128^2 latent ----
    B = 34
    x = torch.randn(B, 4, 128, 128, device="cuda")
    cond = {"crossattn": torch.randn(B, 77, 2048, device="cuda"), "vector": torch.randn(B, 2816, device="cuda"),
            "control": torch.randn(B, 4, 128, 128, device="cuda")}
    t = torch.full((B,), 500.0, device="cuda")
    call_args = (x, t, cond)
    calls = {"bf16": [], "fp8": []}
    res["resident_bytes"] = {}
    for rep in range(3):
        for mode in ("bf16", "fp8"):
            set_mode(net, mode)
            res["resident_bytes"][mode] = packed_bytes(net)
            ms, clk = time_call(net, call_args, args.reps)
            calls[mode].append({"ms": ms, "sm_mhz": clk.get("sm_mhz"), "reasons": clk.get("reasons")})
            if mode == "fp8" and rep == 2:
                res["fp8_shape_table"] = shape_table(net)
            if mode == "bf16" and rep == 2:
                res["bf16_shape_table"] = shape_table(net)
    res["call_34rows_128"] = {k: {"median_ms": float(np.median([c["ms"] for c in v])), "windows": v} for k, v in calls.items()}
    # ---- 3. the cfg3 EDM step (no VAE: a random latent) ----
    from supir_b200 import sampling
    latent = w["in_px"] * w["upscale"] // 8
    c = {"crossattn": torch.randn(1, 77, 2048, device="cuda"), "vector": torch.randn(1, 2816, device="cuda")}
    uc = {"crossattn": torch.randn(1, 77, 2048, device="cuda"), "vector": torch.randn(1, 2816, device="cuda")}
    z = 0.5 * torch.randn(1, 4, latent, latent, device="cuda")
    steps = {"bf16": [], "fp8": []}
    for rep in range(3):
        for mode in ("bf16", "fp8"):
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
    short = {k: v for k, v in res.items() if not k.endswith("shape_table")}
    short["fp8_shape_table_top"] = res["fp8_shape_table"]["rows"][:12]
    print(json.dumps(short))


if __name__ == "__main__":
    main()
