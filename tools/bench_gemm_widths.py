"""Per-width timing of every GEMM / implicit-GEMM conv shape of one denoiser call (GLVControl + LightGLVUNet, full SDXL
depth, random weights), the data `pick_bn`'s cost constants are fitted to.

One eager pass over the captured plan records each GEMM-class launch with its operands. Every distinct launch signature is
then replayed at each forced tile width (`supir_set_gemm_tile_n`) and at the automatic choice, `--reps` launches between a
CUDA-event pair after `--warmup` launches. The table gives the mean ms per launch, the launch count per call, whether the
launch can take the staged (TMA) epilogue, and the width the automatic choice takes.

    python tools/bench_gemm_widths.py [--B 34] [--latent 128] [--dtype bf16|fp16] [--reps 10] [--json out.json]

`--ksweep` instead times the step's short-k-loop signatures (bias + residual, folded LayerNorm without residual, a conv3x3
with a per-image vector) at several K and fits t = a + b K per signature and width: 1 / b is the k-loop's rate, `a` the
K-independent cost of a launch (epilogue, pipeline fill, tile restarts), and `a` over the tiles per CTA the fixed cost of one
tile. It prints the card, its power limit and the median SM clock of the sweep.

    python tools/bench_gemm_widths.py --ksweep [--widths 128,160] [--reps 30] [--json out.json]
"""
import argparse
import json
import math
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import ClockSampler  # noqa: E402
from supir_b200 import _native, nets, ops, wrappers  # noqa: E402

CFG = dict(adm_in_channels=2816, num_classes="sequential", use_checkpoint=True, in_channels=4, out_channels=4,
           model_channels=320, attention_resolutions=[4, 2], num_res_blocks=2, channel_mult=[1, 2, 4], num_head_channels=64,
           use_spatial_transformer=True, use_linear_in_transformer=True, transformer_depth=[1, 2, 10], context_dim=2048,
           spatial_transformer_attn_type="softmax-xformers", legacy=False)
WIDTHS = (64, 128, 160, 256)


def _al16(t):
    return t is None or (t.data_ptr() % 16 == 0 and (t.dim() < 2 or t.stride(0) % 8 == 0))


def record_launches(w):
    """(signature, replay closure, stageable) of every GEMM-class launch of one eager pass over the largest plan."""
    rec = []
    wrapped = {}

    def wrap(name, f, sig):
        def g(*a, **kw):
            out = sig(*a, **kw)
            rec.append(out + (lambda: f(*a, **kw),))
            return f(*a, **kw)
        wrapped[name] = f
        setattr(ops, name, g)

    def stage_ok(out, res):
        return out.dtype != torch.float32 and _al16(out) and _al16(res)

    wrap("gemm", ops.gemm, lambda a, w_, out, **kw: (
        ("gemm", a.shape[0], w_.shape[0], a.shape[1], kw.get("act", 0), kw.get("residual") is not None),
        stage_ok(out, kw.get("residual"))))
    wrap("conv3x3", ops.conv3x3, lambda x, B, H, W, wp, out, **kw: (
        ("conv3x3", x.shape[0], wp.shape[0], wp.shape[1], kw.get("act", 0), kw.get("residual") is not None),
        stage_ok(out, kw.get("residual"))))
    wrap("conv_geom", ops.conv_geom, lambda x, B, Hin, Win, wp, out, geom, **kw: (
        ("conv_geom", B * geom["Hout"] * geom["Wout"], wp.shape[0], wp.shape[1], kw.get("act", 0), False),
        stage_ok(out, None)))
    plan = w._plans[max(w._plans, key=lambda k: k[0])]
    try:
        plan._run()
        torch.cuda.synchronize()
    finally:
        for n, f in wrapped.items():
            setattr(ops, n, f)
    return rec


def time_launch(fn, lib, bn, warmup, reps):
    lib.supir_set_gemm_tile_n(bn)
    try:
        for _ in range(warmup):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
    finally:
        lib.supir_set_gemm_tile_n(0)
    return e0.elapsed_time(e1) / reps


# (name, kind, M or (B, H, W), N, epilogue, K values, K of the step): the cooperative-width signatures of one 34-row
# denoiser call whose k-loop is short, swept over K up to 2 x the step's value (conv: K = 9 Cin). The fit is only as good as
# the line, so the time at the step's own K is printed beside it.
KSWEEP = (
    ("res 33792x1280", "gemm", 33792, 1280, "bias+res", (640, 1280, 1920, 2560), 1280),
    ("res 135168x640", "gemm", 135168, 640, "bias+res", (320, 640, 960, 1280), 640),
    ("ln 33792x3840", "gemm", 33792, 3840, "ln+bias", (640, 1280, 1920, 2560), 1280),
    ("ln 135168x1920", "gemm", 135168, 1920, "ln+bias", (320, 640, 960, 1280), 640),
    ("conv 33x64x64->640", "conv", (33, 64, 64), 640, "bias+rowvec", (2304, 3456, 4608, 5760), 5760),
)


def _ksweep_launch(kind, M, N, K, epi, dtype):
    g = torch.Generator(device="cuda").manual_seed(K)
    rn = lambda *s: torch.randn(*s, generator=g, device="cuda")  # noqa: E731
    if kind == "conv":
        B, H, W = M
        x, wp = rn(B * H * W, K // 9).to(dtype), (rn(N, K) / math.sqrt(K)).to(dtype)
        out, bias, rv = torch.empty(B * H * W, N, dtype=dtype, device="cuda"), rn(N), rn(B, N)
        return lambda: ops.conv3x3(x, B, H, W, wp, out, bias=bias, rowvec=rv), B * H * W, (B * math.ceil(H / 8) * math.ceil(W / 16))
    a, w = rn(M, K).to(dtype), (rn(N, K) / math.sqrt(K)).to(dtype)
    out, bias = torch.empty(M, N, dtype=dtype, device="cuda"), rn(N)
    res = rn(M, N).to(dtype) if "res" in epi else None
    ln = (torch.stack([rn(M).abs() + 0.5, rn(M)], 1).contiguous(), rn(N)) if "ln" in epi else None
    return lambda: ops.gemm(a, w, out, bias=bias, residual=res, ln=ln), M, math.ceil(M / 128)


def ksweep(args, lib, dtype):
    """Fit t = a + b K per (signature, width); see the module docstring."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    try:
        name_pl = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                 capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        name_pl = "nvidia-smi unavailable"
    widths = [int(x) for x in args.widths.split(",")]
    clocks = ClockSampler(0)
    clocks.start()
    rows = []
    try:
        for sig, kind, M, N, epi, ks, step_k in KSWEEP:
            t = {bn: [] for bn in widths}
            for K in ks:
                fn, rows_m, m_tiles = _ksweep_launch(kind, M, N, K, epi, dtype)
                for bn in widths:
                    t[bn].append(time_launch(fn, lib, bn, args.warmup, args.reps))
            for bn in widths:
                b, a = np.polyfit(np.array(ks, float), np.array(t[bn]) * 1e-3, 1)
                tiles_per_cta = math.ceil(m_tiles * math.ceil(N / bn) / sms)
                r = {"sig": sig, "epilogue": epi, "M": rows_m, "N": N, "bn": bn, "K": list(ks), "ms": [round(v, 4) for v in t[bn]],
                     "kloop_tflops": 2.0 * rows_m * N / b / 1e12, "a_us": a * 1e6, "tiles_per_cta": tiles_per_cta,
                     "a_per_tile_us": a * 1e6 / tiles_per_cta, "step_K": step_k, "step_K_us": t[bn][ks.index(step_k)] * 1e3}
                rows.append(r)
                print(f"{sig:20s} {epi:12s} bn {bn:3d}  " + " ".join(f"K {k}: {v * 1e3:7.1f} us" for k, v in zip(ks, t[bn]))
                      + f"  | k-loop {r['kloop_tflops']:5.0f} TFLOP/s, a {r['a_us']:6.1f} us, {tiles_per_cta} tiles/CTA, "
                      f"a per tile {r['a_per_tile_us']:5.2f} us | at the step's K {step_k}: {r['step_K_us']:7.1f} us", flush=True)
    finally:
        clk = clocks.stop()
    print(f"# {torch.cuda.get_device_name(0)} ({name_pl}), {args.dtype}, {sms} SMs, median SM clock {clk.get('sm_mhz')} MHz, "
          f"throttle reasons {clk.get('reasons')}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"device": name_pl, "dtype": args.dtype, "clocks": clk, "rows": rows}, f, indent=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=34, help="network batch (windows x CFG pair); the bench's largest call is 34")
    ap.add_argument("--latent", type=int, default=128)
    ap.add_argument("--dtype", choices=["bf16", "fp16"], default="bf16")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--json", default=None)
    ap.add_argument("--ksweep", action="store_true", help="K sweep of the short-k-loop signatures instead of the call's table")
    ap.add_argument("--widths", default="128,160", help="--ksweep: forced tile widths")
    args = ap.parse_args()
    dtype = {"bf16": torch.bfloat16, "fp16": torch.float16}[args.dtype]
    lib = _native.load()
    if args.ksweep:
        return ksweep(args, lib, dtype)
    with torch.device("cuda"):
        unet = nets.LightGLVUNet(mode="XL-base", project_type="ZeroSFT", project_channel_scale=2, **CFG).to(dtype)
        ctrl = nets.GLVControl(input_upscale=1, **CFG).to(dtype)
    w = wrappers.ControlWrapper(unet, dtype=dtype)
    w.load_control_model(ctrl)
    w.pack()
    B, hw = args.B, args.latent
    x = torch.randn(B, 4, hw, hw, device="cuda")
    c = {"control": torch.randn(B, 4, hw, hw, device="cuda"), "crossattn": torch.randn(B, 77, 2048, device="cuda"),
         "vector": torch.randn(B, 2816, device="cuda")}
    w(x, torch.full((B,), 500, device="cuda"), c, 1.0)
    torch.cuda.synchronize()
    rec = record_launches(w)
    shapes = {}
    for sig, staged, fn in rec:
        s = shapes.setdefault(sig, {"count": 0, "staged": staged, "fn": fn})
        s["count"] += 1
        s["staged"] = s["staged"] and staged
    dev = torch.cuda.get_device_name(0)
    print(f"# {dev}, B={B}, latent {hw}, {args.dtype}, {len(rec)} GEMM-class launches, {len(shapes)} signatures; "
          f"{sum(1 for _, st, _ in rec if not st)} launches cannot take the staged epilogue")
    print(f"{'op':9s} {'M':>7s} {'N':>6s} {'K':>6s} act res  n  staged " + " ".join(f"{b:>8d}" for b in WIDTHS) + "     auto  best")
    rows = []
    for sig, s in sorted(shapes.items(), key=lambda kv: -kv[1]["count"] * 2.0 * kv[0][1] * kv[0][2] * kv[0][3]):
        t = {bn: time_launch(s["fn"], lib, bn, args.warmup, args.reps) for bn in WIDTHS}
        auto = time_launch(s["fn"], lib, 0, args.warmup, args.reps)
        best = min(t, key=t.get)
        rows.append({"op": sig[0], "M": sig[1], "N": sig[2], "K": sig[3], "act": sig[4], "residual": sig[5], "count": s["count"],
                     "staged": s["staged"], "ms": {str(k): round(v, 4) for k, v in t.items()}, "auto_ms": round(auto, 4), "best": best})
        print(f"{sig[0]:9s} {sig[1]:7d} {sig[2]:6d} {sig[3]:6d} {sig[4]:3d} {int(sig[5]):3d} {s['count']:3d} {str(s['staged']):>7s} "
              + " ".join(f"{t[b]:8.3f}" for b in WIDTHS) + f" {auto:8.3f}  {best}", flush=True)
    tot = {bn: sum(r["count"] * r["ms"][str(bn)] for r in rows) for bn in WIDTHS}
    tot_auto = sum(r["count"] * r["auto_ms"] for r in rows)
    tot_best = sum(r["count"] * min(r["ms"].values()) for r in rows)
    print("# per-call totals (ms): " + ", ".join(f"{b}: {tot[b]:.1f}" for b in WIDTHS) + f", auto: {tot_auto:.1f}, best per shape: {tot_best:.1f}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"device": dev, "B": B, "latent": hw, "dtype": args.dtype, "rows": rows, "total_auto_ms": tot_auto,
                       "total_best_ms": tot_best}, f, indent=1)


if __name__ == "__main__":
    main()
