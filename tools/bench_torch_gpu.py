"""The reference's OWN GPU path timed on the same GPU next to supir_b200 (SURVEY.md §8d last row, BASELINE.md §4 item 3: "the real
competitor"): the oracle — a functional restatement of GLVControl + LightGLVUNet that calls exactly the torch ops the
reference's modules call (F.linear / F.conv2d / F.group_norm / F.layer_norm / F.scaled_dot_product_attention) — run on
`cuda` under `torch.autocast(bfloat16)` with bf16 weights (test.py --loading_half_params --diff_dtype bf16), eager mode like the
reference (cuBLAS / cuDNN / flash-attention kernels, no CUDA graph). With `--dtype fp16` both sides compute in fp16 instead:
ControlWrapper(dtype=float16) against the oracle under `torch.autocast(float16)` with fp16 weights (test.py's default,
--diff_dtype fp16).

    python tools/bench_torch_gpu.py [latent_side=128] [batches=2,14,98] [--dtype bf16|fp16]

Prints one JSON line per batch with ms per denoiser call for both implementations on the same inputs, the SM clock
(nvidia-smi, sampled during each timed window) and the relative Frobenius difference of their outputs. TOOL ONLY: nothing here is on the product path (the product never imports oracle/).
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import bench  # noqa: E402


def time_ms(fn, warmup=2, iters=5, clocks=None):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    if clocks is not None:
        clocks.mark()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    argv = list(sys.argv[1:])
    dname = "bf16"
    if "--dtype" in argv:
        i = argv.index("--dtype")
        dname = argv[i + 1]
        del argv[i:i + 2]
    dtype = {"bf16": torch.bfloat16, "fp16": torch.float16}[dname]
    side = int(argv[0]) if len(argv) > 0 else 128
    batches = [int(b) for b in (argv[1] if len(argv) > 1 else "2,14,98").split(",")]
    from oracle import unet as ounet
    from supir_b200 import nets, wrappers
    sd = bench.oracle_state_dict(fast=True)
    with torch.device("meta"):
        unet = nets.LightGLVUNet(mode="XL-base", project_type="ZeroSFT", project_channel_scale=2, **bench.UNET_CFG)
        ctrl = nets.GLVControl(input_upscale=1, **bench.UNET_CFG)
    w = wrappers.ControlWrapper(unet, dtype=dtype)
    w.load_control_model(ctrl)
    w.to_empty(device="cuda")
    w.load_state_dict(sd, strict=True)
    sd_gpu = {k: v.to("cuda", dtype) for k, v in sd.items()}
    del sd
    torch.set_default_device("cuda")          # the oracle creates its small constants (timestep frequencies) on the default device
    flop = bench.flop_denoiser(side)

    def timed(fn):
        cs = bench.ClockSampler(torch.cuda.current_device())
        cs.start()
        ms = time_ms(fn, clocks=cs)
        return ms, cs.stop()
    for B in batches:
        g = torch.Generator(device="cuda").manual_seed(B)
        x = torch.randn(B, 4, side, side, generator=g)
        cond = {"control": torch.randn(B, 4, side, side, generator=g), "crossattn": torch.randn(B, 77, 2048, generator=g),
                "vector": torch.randn(B, 2816, generator=g)}
        t = torch.full((B,), 500, dtype=torch.long)
        line = {"latent": side, "batch": B, "dtype": dname, "gpu": torch.cuda.get_device_name(), "tflop_per_call": flop * B / 2 / 1e12}
        key = f"torch_eager_{dname}_ms"
        try:
            def ref():
                with torch.no_grad(), torch.autocast("cuda", dtype=dtype):
                    return ounet.control_wrapper_forward(sd_gpu, x, t, cond, 1.0)
            out_ref = ref().float()
            line[key], line["torch_clocks"] = timed(ref)
            line["torch_tflops"] = flop * B / 2 / (line[key] * 1e-3) / 1e12
            line["torch_peak_mem_gib"] = torch.cuda.max_memory_allocated() / 2 ** 30
        except torch.OutOfMemoryError as e:      # eager PyTorch keeps every intermediate of the call alive in the caching allocator
            out_ref = None
            line[key] = None
            line["torch_error"] = "out of memory: " + str(e)[:120]
            torch.cuda.empty_cache()
        out = w(x, t, cond, control_scale=1.0)
        line["supir_b200_ms"], line["supir_clocks"] = timed(lambda: w(x, t, cond, control_scale=1.0))
        line["supir_tflops"] = flop * B / 2 / (line["supir_b200_ms"] * 1e-3) / 1e12
        if out_ref is not None:
            line["speedup"] = line[key] / line["supir_b200_ms"]
            line["rel_fro_between_them"] = float((out - out_ref).norm() / out_ref.norm())
        print(json.dumps(line), flush=True)
        w.invalidate()
        del out, out_ref
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()


if __name__ == "__main__":
    main()
