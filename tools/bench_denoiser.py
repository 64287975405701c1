"""Quick timing of one denoiser network call (GLVControl + LightGLVUNet, full SDXL depth) on random weights."""
import sys, os, time, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from supir_b200 import nets, wrappers, _native

CFG = dict(adm_in_channels=2816, num_classes="sequential", use_checkpoint=True, in_channels=4, out_channels=4,
           model_channels=320, attention_resolutions=[4, 2], num_res_blocks=2, channel_mult=[1, 2, 4], num_head_channels=64,
           use_spatial_transformer=True, use_linear_in_transformer=True, transformer_depth=[1, 2, 10], context_dim=2048,
           spatial_transformer_attn_type="softmax-xformers", legacy=False)
FLOP = {64: 4.766e12, 128: 20.292e12, 256: 107.887e12}

def record_shapes(path):
    """Wrap ops.gemm / ops.conv3x3 to log the launch order of GEMM-class kernels (joined offline with an ncu launch list)."""
    from supir_b200 import ops
    log = []
    og, oc = ops.gemm, ops.conv3x3

    def gemm(a, w, out, **kw):
        log.append(["gemm", a.shape[0], w.shape[0], a.shape[1], kw.get("act", 0), kw.get("residual") is not None])
        return og(a, w, out, **kw)

    def conv(x, B, H, W, wp, out, **kw):
        log.append(["conv3x3", x.shape[0], wp.shape[0], wp.shape[1], kw.get("act", 0), kw.get("residual") is not None])
        return oc(x, B, H, W, wp, out, **kw)
    ops.gemm, ops.conv3x3 = gemm, conv
    import atexit
    atexit.register(lambda: json.dump(log, open(path, "w")))


def breakdown(w, B, hw):
    """Per-op device time of one eager pass over the captured plan: every supir_b200.ops launch between a CUDA-event pair."""
    import inspect, collections
    from supir_b200 import ops
    names = [n for n, f in vars(ops).items() if inspect.isfunction(f) and f.__module__ == ops.__name__ and not n.startswith("_")
             and n not in ("groupnorm_ws_size", "upsample2x_conv3x3", "conv3x3_stride2", "fold_upsample_weights", "fold_layernorm")]
    rec, orig = [], {}
    for n in names:
        f = orig[n] = getattr(ops, n)

        def wrap(*a, _f=f, _n=n, **kw):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = _f(*a, **kw)
            e1.record()
            key = _n
            if _n == "attention":      # q [B*Lq, H*64], k [B*Lk, H*64]: split self- from cross-attention and by level
                key = f"attention q{tuple(a[0].shape)} k{tuple(a[1].shape)}"
            rec.append((key, e0, e1))
            return r
        setattr(ops, n, wrap)
    plan = w._plans[max(w._plans, key=lambda k: k[0])]
    try:
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        plan._run()
        t1.record()
        torch.cuda.synchronize()
    finally:
        for n, f in orig.items():
            setattr(ops, n, f)
    agg = collections.Counter()
    cnt = collections.Counter()
    for n, e0, e1 in rec:
        agg[n] += e0.elapsed_time(e1)
        cnt[n] += 1
    tot = sum(agg.values())
    print(f"== eager pass B={B} latent={hw}: wall {t0.elapsed_time(t1):.1f} ms, sum of op times {tot:.1f} ms, {len(rec)} calls")
    for n, t in agg.most_common():
        print(f"   {n:24s} {t:9.2f} ms {100*t/tot:5.1f}%  n={cnt[n]}")


def main():
    if os.environ.get("BENCH_SHAPE_LOG"):
        record_shapes(os.environ["BENCH_SHAPE_LOG"])
    argv = list(sys.argv[1:])
    dtype = torch.bfloat16
    if "--dtype" in argv:           # --dtype bf16 | fp16: the compute dtype of the networks
        i = argv.index("--dtype")
        dtype = {"bf16": torch.bfloat16, "fp16": torch.float16}[argv[i + 1]]
        del argv[i:i + 2]
    sizes = [int(a) for a in argv] or [64, 128]
    t0 = time.time()
    with torch.device("cuda"):
        # parameters held in the compute dtype (half the memory of fp32): packing then rounds nothing further
        unet = nets.LightGLVUNet(mode="XL-base", project_type="ZeroSFT", project_channel_scale=2, **CFG).to(dtype)
        ctrl = nets.GLVControl(input_upscale=1, **CFG).to(dtype)
    w = wrappers.ControlWrapper(unet, dtype=dtype)
    w.load_control_model(ctrl)
    w.pack()
    torch.cuda.synchronize()
    print(f"build+pack {time.time()-t0:.1f}s, mem {torch.cuda.memory_allocated()/2**30:.1f} GiB", flush=True)
    for hw in sizes:
        for B in [int(b) for b in os.environ.get('BENCH_B', '2,4,8').split(',')]:
            if hw >= 256 and B > 2:
                continue
            x = torch.randn(B, 4, hw, hw, device="cuda")
            c = {"control": torch.randn(B, 4, hw, hw, device="cuda"), "crossattn": torch.randn(B, 77, 2048, device="cuda"),
                 "vector": torch.randn(B, 2816, device="cuda")}
            t = torch.full((B,), 500, device="cuda")
            _native.reset_launch_count()
            out = w(x, t, c, 1.0)
            torch.cuda.synchronize()
            launches = _native.launch_count() // 2   # warm-up + capture
            for _ in range(2):
                w(x, t, c, 1.0)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            iters = 5
            e0.record()
            for _ in range(iters):
                w(x, t, c, 1.0)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / iters
            fl = FLOP.get(hw, 0) * B / 2
            if os.environ.get("BENCH_BREAKDOWN") == "1":
                breakdown(w, B, hw)
            print(json.dumps({"latent": hw, "B": B, "ms": round(ms, 3), "tflops": round(fl / ms / 1e9, 1), "launches": launches,
                              "finite": bool(torch.isfinite(out).all()), "mem_gib": round(torch.cuda.max_memory_allocated() / 2**30, 1)}), flush=True)

main()
