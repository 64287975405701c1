"""GPU tests of the fp16 compute mode (the `_f16` entry points and ControlWrapper(dtype=torch.float16)).

Per op: every `_f16` entry point the diffusion networks call, against fp32 PyTorch on the same fp16-rounded inputs, with
outputs written into NaN-filled buffers. Each case must meet |err| <= 4e-3 + 4e-3 |ref| per element, and its relative
Frobenius error must be at most 1/4 of the bf16 entry point's on the same inputs: fp16 carries 3 more mantissa bits than
bf16, so a kernel that silently computed or stored bf16 would fail the ratio.

Networks: the full-width depth-1 GLVControl + LightGLVUNet of unet_fullwidth_depth1.npz against the fp32 oracle, the real
SUPIR-v0 layout on one 128^2 latent window, graph replay against an eager run of the same plan, bf16 <-> fp16 switching,
SUPIRModel(diffusion_dtype="fp16") through batchify_sample (untiled and tiled), and the sharded sampler in fp16 (>= 2 GPUs).
"""
import json
import math
import os
import warnings

import numpy as np
import pytest
import torch

from weights import make_state_dict, randn

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
H16, BF = torch.float16, torch.bfloat16
SENTINEL = 7.0


def _ops():
    from supir_b200 import _native, ops
    return ops, _native


def _master(shape, seed, scale=1.0):
    """fp32 values that are exact in fp16 (the common input of the fp16 and bf16 runs)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale).half().float()


def _rel(a, b):
    return float((a.float() - b).norm() / b.norm())


def _check(got, ref, what, atol=4e-3, rtol=4e-3):
    g = got.float()
    assert bool(torch.isfinite(g).all()), f"{what}: {int((~torch.isfinite(g)).sum())} non-finite (unwritten?) elements"
    err = (g - ref).abs()
    nbad = int((err > atol + rtol * ref.abs()).sum())
    assert nbad == 0, f"{what}: {nbad} elements out of tolerance, max err {float(err.max()):.4g}"


def _compare(run, ref, what):
    """run(dtype) -> output of the op with all 16-bit operands in `dtype`; checks the fp16 result and the 1/4 ratio."""
    o16, obf = run(H16), run(BF)
    _check(o16, ref, what)
    e16, ebf = _rel(o16, ref), _rel(obf, ref)
    assert e16 <= 0.25 * ebf, f"{what}: fp16 rel error {e16:.3g} is not below 1/4 of bf16's {ebf:.3g}"
    return o16


class _Out:
    """A [rows, cols] output view inside a wider buffer: the view starts NaN, eight columns on each side (16 bytes of 16-bit
    values, which keeps the vectorised stores aligned) hold SENTINEL."""

    def __init__(self, rows, cols, dtype):
        self.buf = torch.full((rows, cols + 16), SENTINEL, dtype=dtype, device="cuda")
        self.view = self.buf[:, 8:8 + cols]
        self.view.fill_(float("nan"))

    def done(self):
        side = torch.cat([self.buf[:, :8], self.buf[:, -8:]], 1).float()
        assert bool((side == SENTINEL).all()), "write outside the output view"
        return self.view


def _gelu(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


# ---------------------------------------------------------------------------------------------------------------------
# GEMM epilogues at every tile width, ragged M / N, persistent tile count of SMs + 1
# ---------------------------------------------------------------------------------------------------------------------
EPILOGUES = ["plain", "bias", "rowvec", "ln", "silu", "geglu", "residual", "f32"]


@pytest.mark.parametrize("bn", [64, 128, 160, 256])
@pytest.mark.parametrize("epi", EPILOGUES)
def test_gemm_f16_epilogues(epi, bn):
    ops, native = _ops()
    lib = native.load()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    K = 320
    N = 2 * bn * 2 + 32 if epi == "geglu" else bn * 2 + 24          # ragged N (GEGLU: multiple of 32)
    M = (sms + 1) * 128 // (N // bn + 1) + 77                          # ~SMs + 1 tiles, ragged M
    a = _master((M, K), 1)
    w = _master((N, K), 2, K ** -0.5)
    bias = _master((N,), 3, 0.5)
    rows_per_batch = M // 3 + 5
    rowvec = _master((3, N), 4, 0.5)
    ncol = N // 2 if epi == "geglu" else N
    res = _master((M, ncol), 5)
    gamma, beta = 1.0 + 0.1 * _master((K,), 6), 0.1 * _master((K,), 7)
    kw, ref = {}, a @ w.t()
    if epi == "bias":
        kw, ref = dict(bias=bias), ref + bias
    elif epi == "rowvec":
        rv = torch.repeat_interleave(rowvec, rows_per_batch, 0)[:M]
        kw, ref = dict(rowvec=rowvec, rows_per_batch=rows_per_batch), ref + rv
    elif epi == "silu":
        kw, ref = dict(bias=bias, act=1), torch.nn.functional.silu(ref + bias)
    elif epi == "geglu":
        y = ref + bias
        yv = y.view(M, -1, 2, 16)
        ref = (yv[:, :, 0] * _gelu(yv[:, :, 1])).reshape(M, ncol)
        kw = dict(bias=bias, act=2)
    elif epi == "residual":
        kw, ref = dict(bias=bias, residual=res), ref + bias + res
    elif epi == "ln":
        an = torch.nn.functional.layer_norm(a, (K,), gamma, beta, 1e-5)
        ref = an @ w.t() + bias

    def run(dt):
        o = _Out(M, ncol, torch.float32 if epi == "f32" else dt)
        args = dict(kw)
        if "residual" in args:
            args["residual"] = res.to(dt)
        A, W = a.to(dt), w
        if epi == "ln":
            wg, colsum, b2 = ops.fold_layernorm(w, bias, gamma, beta, dtype=dt)
            st = torch.empty((M, 2), dtype=torch.float32, device="cuda")
            ops.layernorm_stats(A, st)
            args = dict(bias=b2, ln=(st, colsum))
            W = wg
        lib.supir_set_gemm_tile_n(bn)
        try:
            ops.gemm(A, W.to(dt), o.view, **args)
        finally:
            lib.supir_set_gemm_tile_n(0)
        return o.done()

    _compare(run, ref, f"gemm {epi} bn={bn}")


def test_gemm_f16_overflow_matches_torch_cast():
    """Results beyond the fp16 range become +-inf exactly where torch's cast of the fp32 product puts them."""
    ops, _ = _ops()
    M, N, K = 300, 200, 256
    a = _master((M, K), 11)
    w = _master((N, K), 12, 40.0)            # |a.w| ~ 640 * N(0,1) ... scaled up below to straddle 65504
    a[::7] *= 150.0
    a = a.half().float()
    exact = a @ w.t()
    assert bool((exact.abs() > 65504).any()) and bool((exact.abs() < 60000).any())
    out = torch.full((M, N), float("nan"), dtype=H16, device="cuda")
    ops.gemm(a.half(), w.half(), out)
    want = exact.half()
    assert torch.equal(torch.isinf(out), torch.isinf(want))
    assert torch.equal(torch.sign(out[torch.isinf(out)]), torch.sign(want[torch.isinf(want)]))


# ---------------------------------------------------------------------------------------------------------------------
# convolutions
# ---------------------------------------------------------------------------------------------------------------------
def _nhwc(x):
    B, C, H, W = x.shape
    return x.permute(0, 2, 3, 1).reshape(B * H * W, C).contiguous()


@pytest.mark.parametrize("kind", ["conv3x3", "stride2", "upsample"])
def test_conv_f16(kind):
    ops, _ = _ops()
    from supir_b200 import nets
    F = torch.nn.functional
    B, Cin, Cout, H, W = 2, 64, 96, 19, 23
    x = _master((B, Cin, H, W), 21)
    w = _master((Cout, Cin, 3, 3), 22, (9 * Cin) ** -0.5).half().float()
    bias = _master((Cout,), 23, 0.5)
    if kind == "conv3x3":
        ref = F.conv2d(x, w, bias, padding=1)
    elif kind == "stride2":
        ref = F.conv2d(x, w, bias, stride=2, padding=1)
    else:
        ref = F.conv2d(F.interpolate(x, scale_factor=2, mode="nearest"), w, bias, padding=1)
    Ho, Wo = ref.shape[2], ref.shape[3]
    ref = _nhwc(ref)

    def run(dt):
        xs = _nhwc(x).to(dt)
        o = _Out(B * Ho * Wo, Cout, dt)
        if kind == "conv3x3":
            ops.conv3x3(xs, B, H, W, nets.pack_conv3x3(w, dt), o.view, bias=bias)
        elif kind == "stride2":
            ops.conv3x3_stride2(xs, B, H, W, nets.pack_conv3x3(w, dt), o.view, 1, bias=bias)
        else:
            ops.upsample2x_conv3x3(xs, B, H, W, ops.fold_upsample_weights(w, dt), o.view, bias=bias)
        return o.done()

    # the sub-pixel taps are sums of up to four weights rounded once to the storage type: compare against those sums
    _compare(run, ref, f"conv {kind}")


@pytest.mark.parametrize("large", [False, True])
def test_small_convs_f16(large):
    """Entry conv (Cin = 4, direct kernel or im2col + GEMM) with a residual, exit conv (Cout = 4, direct or on the tensor
    cores + the NHWC crop exit)."""
    ops, _ = _ops()
    from supir_b200 import ops as O
    F = torch.nn.functional
    pool = O.Pool()
    H = W = 128 if large else 24
    B, Cin, C = 2, 4, 64
    x = _master((B, Cin, H, W), 31)
    w = _master((C, Cin, 3, 3), 32, 0.2).half().float()
    bias = _master((C,), 33, 0.2).half().float()
    res = _master((B * H * W, C), 34)
    ref = _nhwc(F.conv2d(x, w, bias, padding=1)) + res

    def run_in(dt):
        o = _Out(B * H * W, C, dt)
        ops.conv3x3_small_cin(x, w, bias, o.view, residual=res.to(dt), w_packed=O.pack_small_cin_weight(w, dt) if large else None,
                              pool=pool if large else None)
        return o.done()

    _compare(run_in, ref, f"small-Cin conv {H}")
    h = _master((B * H * W, C), 35)
    wo = _master((4, C, 3, 3), 36, (9 * C) ** -0.5).half().float()
    bo = _master((4,), 37, 0.2).half().float()
    ref_o = F.conv2d(h.view(B, H, W, C).permute(0, 3, 1, 2), wo, bo, padding=1)

    def run_out(dt):
        out = torch.full((B, 4, H, W), float("nan"), device="cuda")
        ops.conv3x3_small_cout(h.to(dt), B, H, W, wo.permute(0, 2, 3, 1).contiguous(), bo, out,
                               packed=O.pack_small_cout_weight(wo, bo, dt) if large else None, pool=pool if large else None)
        return out

    _compare(run_out, ref_o, f"small-Cout conv {H}")


# ---------------------------------------------------------------------------------------------------------------------
# attention
# ---------------------------------------------------------------------------------------------------------------------
def _ref_attention(q, k, v, B, H, Lq, Lk, scale):
    qh = q.view(B, Lq, H, 64).transpose(1, 2)
    kh = k.view(B, Lk, H, 64).transpose(1, 2)
    vh = v.view(B, Lk, H, 64).transpose(1, 2)
    p = torch.softmax(qh @ kh.transpose(-1, -2) * scale, dim=-1)
    return (p @ vh).transpose(1, 2).reshape(B * Lq, H * 64)


@pytest.mark.parametrize("Lk", [77, 1024, 4096])
@pytest.mark.parametrize("logits", ["random", "rising"])
def test_attention_f16(Lk, logits):
    ops, _ = _ops()
    B, H, Lq = 2, 5, 300
    C = H * 64
    if logits == "random":
        q, k, v = _master((B * Lq, C), 41, 1.5), _master((B * Lk, C), 42, 1.5), _master((B * Lk, C), 43)
    else:
        # key block j aligned with the queries with a gain growing with j: the row maximum rises in every 128-key block
        g = torch.Generator(device="cuda").manual_seed(44)
        q = torch.randn((B, Lq, H, 64), generator=g, device="cuda")
        qdir = q / q.norm(dim=-1, keepdim=True)
        u = qdir[:, 0::2].mean(dim=1, keepdim=True)
        u = u / u.norm(dim=-1, keepdim=True)
        q = qdir * 8.0
        q[:, 0::2] = u * 8.0 + 0.05 * q[:, 0::2]
        blocks = (torch.arange(Lk, device="cuda") // 128).float().view(1, Lk, 1, 1)
        k = torch.randn((B, Lk, H, 64), generator=g, device="cuda") * 0.3 + u * (blocks * 6.3 / (8.0 * 0.125))
        v = torch.randn((B, Lk, H, 64), generator=g, device="cuda")
        q, k, v = (t.reshape(-1, C).half().float() for t in (q, k, v))
    ref = _ref_attention(q, k, v, B, H, Lq, Lk, 0.125)

    def run(dt):
        o = _Out(B * Lq, C, dt)
        ops.attention(q.to(dt), k.to(dt), v.to(dt), o.view, B, H, Lq, Lk)
        return o.done()

    _compare(run, ref, f"attention Lk={Lk} {logits}")


# ---------------------------------------------------------------------------------------------------------------------
# normalisation, ZeroSFT, axpy, embedding MLP
# ---------------------------------------------------------------------------------------------------------------------
def test_groupnorm_zerosft_layernorm_f16():
    ops, _ = _ops()
    F = torch.nn.functional
    B, HW, C, C1 = 2, 300, 128, 64
    x = _master((B * HW, C), 51, 2.0) + 0.5
    gamma, beta = 1.0 + 0.1 * _master((C,), 52), 0.1 * _master((C,), 53)
    xr = x.view(B, HW, C).permute(0, 2, 1)
    ref_gn = F.silu(F.group_norm(xr, 32, gamma, beta, 1e-5)).permute(0, 2, 1).reshape(B * HW, C)

    def run_gn(dt):
        ws = torch.zeros(ops.groupnorm_ws_size(B, HW, C), dtype=torch.float64, device="cuda")
        ops.groupnorm_stats(x.to(dt), B, HW, ws)
        o = _Out(B * HW, C, dt)
        ops.groupnorm_apply(x.to(dt), B, HW, o.view, gamma, beta, 1e-5, True, sums=ws)
        return o.done()

    _compare(run_gn, ref_gn, "groupnorm + SiLU")

    skip_raw = _master((B * HW, C - C1), 54)
    gb = _master((B * HW, 2 * C), 55, 0.5)
    cs = torch.tensor([0.7], device="cuda")
    hraw = torch.cat([x[:, :C1], skip_raw], 1)
    n = F.group_norm(xr, 32, gamma, beta, 1e-5).permute(0, 2, 1).reshape(B * HW, C)
    ref_sft = (n * (gb[:, :C] + 1.0) + gb[:, C:]) * 0.7 + hraw * 0.3

    def run_sft(dt):
        ws = torch.zeros(ops.groupnorm_ws_size(B, HW, C), dtype=torch.float64, device="cuda")
        ops.groupnorm_stats(x.to(dt), B, HW, ws)
        o = _Out(B * HW, C, dt)
        ops.zerosft_apply(x.to(dt), skip_raw.to(dt), C1, gb.to(dt), o.view, B, HW, ws, gamma, beta, 1e-5, cs)
        return o.done()

    _compare(run_sft, ref_sft, "ZeroSFT")

    ref_ln = F.layer_norm(x, (C,), gamma, beta, 1e-5)

    def run_ln(dt):
        o = _Out(B * HW, C, dt)
        ops.layernorm(x.to(dt), o.view, gamma, beta)
        return o.done()

    _compare(run_ln, ref_ln, "layernorm")
    mean, var = x.mean(1), x.var(1, unbiased=False)
    rstd = torch.rsqrt(var + 1e-5)
    ref_st = torch.stack([rstd, mean * rstd], 1)
    st = torch.empty((B * HW, 2), device="cuda")
    ops.layernorm_stats(x.half(), st)
    _check(st, ref_st, "layernorm stats", atol=1e-4, rtol=1e-4)


def test_axpy_and_linear_small_m_f16():
    ops, _ = _ops()
    F = torch.nn.functional
    a, y = _master((333, 64), 61), _master((333, 64), 62)
    s = torch.tensor([0.37], device="cuda")

    def run_axpy(dt):
        o = _Out(333, 64, dt)
        ops.axpy(a.to(dt), y.to(dt), o.view, s)
        return o.done()

    _compare(run_axpy, a + y * 0.37, "axpy")
    B, N, K = 6, 200, 320
    x = _master((B, K), 63)
    w = _master((N, K), 64, K ** -0.5)
    bias = _master((N,), 65, 0.3).half().float()
    add = _master((B, N), 66)
    ref = F.silu(F.silu(F.silu(x) @ w.t() + bias) + add)

    def run_lin(dt):
        out = torch.full((B, N), float("nan"), device="cuda")
        ops.linear_small_m(x, w.to(dt), bias, out, silu_in=True, silu_out=3, add=add)
        return out

    _compare(run_lin, ref, "linear_small_m")
    xe = _master((1000,), 67, 3.0) * 1.0001       # values between fp16 grid points
    o = torch.empty(1000, dtype=H16, device="cuda")
    ops.f32_to_f16(xe, o)
    assert torch.equal(o, xe.half())


# ---------------------------------------------------------------------------------------------------------------------
# networks
# ---------------------------------------------------------------------------------------------------------------------
def _depth1():
    g = np.load(os.path.join(G, "unet_fullwidth_depth1.npz"))
    cfg = json.loads(str(g["cfg"]))
    return cfg, make_state_dict(json.loads(str(g["shapes"])), seed=31)


def _wrapper(cfg, sd, dtype):
    from supir_b200 import nets, wrappers
    with torch.device("cuda"):
        unet = nets.LightGLVUNet(mode="XL-base", project_type="ZeroSFT", project_channel_scale=2, **cfg)
        ctrl = nets.GLVControl(input_upscale=1, **cfg)
    w = wrappers.ControlWrapper(unet, dtype=dtype)
    w.load_control_model(ctrl)
    w.load_state_dict(sd, strict=True)
    return w


def _inputs(B, side=16):
    x = randn((B, 4, side, side), 41)
    cond = {"control": randn((B, 4, side, side), 42), "crossattn": randn((B, 77, 2048), 43), "vector": randn((B, 2816), 44)}
    t = torch.tensor([950, 120] * (B // 2) + [500] * (B % 2))
    return x, t, cond


def _oracle(sd, x, t, cond, cs):
    from oracle import unet as ounet
    control = ounet.glv_control_forward(sd, cond["control"], t, x, cond["crossattn"], cond["vector"], 320, 64, prefix="control_model.")
    return ounet.light_glv_unet_forward(sd, x, t, cond["crossattn"], cond["vector"], control, cs, 320, 64, prefix="diffusion_model.")


def test_network_parity_f16_vs_oracle_bf16_and_autocast():
    cfg, sd = _depth1()
    x, t, cond = _inputs(2)
    ref = _oracle(sd, x, t, cond, 0.8)
    cc = {k: v.cuda() for k, v in cond.items()}
    w = _wrapper(cfg, sd, torch.float16)
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        o16 = w(x.cuda(), t.cuda(), cc, control_scale=0.8).cpu()
    w.dtype = torch.bfloat16
    obf = w(x.cuda(), t.cuda(), cc, control_scale=0.8).cpu()
    e16, ebf = _rel(o16, ref), _rel(obf, ref)
    print(f"depth-1 networks vs fp32 oracle: fp16 {e16:.4g}, bf16 {ebf:.4g}")
    assert e16 <= 5e-3 and e16 < ebf
    # the reference's default GPU path: the same networks under torch.autocast(float16) with fp16 weights
    sd16 = {k: (v.half() if v.dim() >= 2 else v).cuda() for k, v in sd.items()}
    with torch.device("cuda"), torch.autocast("cuda", dtype=torch.float16):
        ref_ac = _oracle(sd16, x.cuda(), t.cuda(), cc, 0.8).float().cpu()
    a16, abf = _rel(o16, ref_ac), _rel(obf, ref_ac)
    print(f"vs oracle under autocast(float16): fp16 {a16:.4g}, bf16 {abf:.4g}")
    assert a16 < abf


def test_network_f16_batch18_rows():
    cfg, sd = _depth1()
    x, t, cond = _inputs(18, side=8)
    ref = _oracle(sd, x, t, cond, 1.0)
    w = _wrapper(cfg, sd, torch.float16)
    out = w(x.cuda(), t.cuda(), {k: v.cuda() for k, v in cond.items()}, control_scale=1.0).cpu()
    for i in range(18):
        e = _rel(out[i], ref[i])
        assert e <= 1e-2, f"row {i}: rel error {e:.4g}"


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_graph_replay_equals_eager_run(dtype):
    """The captured denoiser call replays exactly what an eager run of the same plan computes, and replays are repeatable."""
    cfg, sd = _depth1()
    x, t, cond = _inputs(2)
    args = (x.cuda(), t.cuda(), {k: v.cuda() for k, v in cond.items()})
    w = _wrapper(cfg, sd, dtype)
    r1 = w(*args, control_scale=0.8).clone()          # builds the plan (eager warm-up + capture) and replays it
    plan = next(iter(w._plans.values()))
    assert plan.graph is not None
    plan.out.fill_(float("nan"))
    plan._run()                                       # the same call, eager: kernel launches, no graph
    torch.cuda.synchronize()
    eager = plan.out.clone()
    r2 = w(*args, control_scale=0.8).clone()          # replay
    assert bool(torch.isfinite(eager).all())
    assert torch.equal(eager, r1) and torch.equal(eager, r2)


def test_f16_dtype_switch_reproduces_each_dtype():
    cfg, sd = _depth1()
    x, t, cond = _inputs(2)
    args = (x.cuda(), t.cuda(), {k: v.cuda() for k, v in cond.items()})
    w = _wrapper(cfg, sd, torch.bfloat16)
    b1 = w(*args, control_scale=0.8).clone()
    w.dtype = torch.float16
    assert not w._packed and not w._plans
    f1 = w(*args, control_scale=0.8).clone()
    f2 = w(*args, control_scale=0.8).clone()
    assert torch.equal(f1, f2)
    assert w.diffusion_model._emb_w.dtype == torch.float16
    w.dtype = torch.bfloat16
    b2 = w(*args, control_scale=0.8)
    assert torch.equal(b1, b2)
    assert not torch.equal(b1, f1)


@pytest.mark.slow
def test_real_layout_f16_one_window():
    """The real SUPIR-v0 layout (full depth and width) on one of the bench's 128^2 latent windows: finite, and within the
    bound test_gpu_bench_networks.py uses for bf16 (3e-2) against the fp32 oracle."""
    import sys
    sys.path.insert(0, os.path.dirname(G[:-len("/golden")]))
    import bench
    from oracle import unet as ounet
    from supir_b200 import nets, wrappers
    sd = bench.oracle_state_dict()
    g = torch.Generator().manual_seed(3)
    for k, v in sd.items():
        if not (k.endswith("weight") and v.dim() >= 2):
            v.add_(0.05 * torch.randn(v.shape, generator=g))
    with torch.device("meta"):
        unet = nets.LightGLVUNet(mode="XL-base", project_type="ZeroSFT", project_channel_scale=2, **bench.UNET_CFG)
        ctrl = nets.GLVControl(input_upscale=1, **bench.UNET_CFG)
    w = wrappers.ControlWrapper(unet, dtype=torch.float16)
    w.load_control_model(ctrl)
    w.to_empty(device="cuda")
    w.load_state_dict(sd, strict=True)
    torch.set_num_threads(min(os.cpu_count() or 1, 64))
    side = 128
    x = randn((1, 4, side, side), 429)
    cond = {"control": randn((1, 4, side, side), 438), "crossattn": randn((1, 77, 2048), 439), "vector": randn((1, 2816), 440)}
    t = torch.tensor([700])
    out = w(x.cuda(), t.cuda(), {k: v.cuda() for k, v in cond.items()}, control_scale=1.0).cpu()
    assert bool(torch.isfinite(out).all())
    ref = ounet.control_wrapper_forward(sd, x, t, cond, 1.0)
    e = _rel(out, ref)
    print(f"real layout fp16 at a {side}^2 latent vs oracle: rel_fro={e:.4g}")
    assert e <= 3e-2
    w.invalidate()
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------------
# the engine end to end, and the sharded sampler
# ---------------------------------------------------------------------------------------------------------------------
class _SeededNoise:
    def __init__(self, base):
        self.base, self.n = base, 0

    def __call__(self, x, **k):
        self.n += 1
        return randn(tuple(x.shape), self.base + self.n).to(x.device, x.dtype)


def _engine(diffusion_dtype, tiled):
    from supir_b200 import model as smodel
    gu = np.load(os.path.join(G, "unet_fullwidth_depth1.npz"))
    gv = np.load(os.path.join(G, "vae_tiny.npz"))
    ucfg, vcfg = json.loads(str(gu["cfg"])), json.loads(str(gv["cfg"]))
    disc = {"target": "sgm.modules.diffusionmodules.discretizer.LegacyDDPMDiscretization"}
    params = {"num_steps": 100, "restore_cfg": 4.0, "s_churn": 0, "s_noise": 1.003, "discretization_config": disc,
              "guider_config": {"target": "sgm.modules.diffusionmodules.guiders.LinearCFG", "params": {"scale": 7.5, "scale_min": 4.0}}}
    sampler = {"target": "sgm.modules.diffusionmodules.sampling.RestoreEDMSampler", "params": params}
    if tiled:
        sampler = {"target": "sgm.modules.diffusionmodules.sampling.TiledRestoreEDMSampler",
                   "params": dict(params, tile_size=16, tile_stride=8, tile_batch=4)}
    cfg = dict(
        control_stage_config={"target": "SUPIR.modules.SUPIR_v0.GLVControl", "params": dict(ucfg, input_upscale=1)},
        network_config={"target": "SUPIR.modules.SUPIR_v0.LightGLVUNet",
                        "params": dict(ucfg, mode="XL-base", project_type="ZeroSFT", project_channel_scale=2)},
        network_wrapper="sgm.modules.diffusionmodules.wrappers.ControlWrapper",
        denoiser_config={"target": "sgm.modules.diffusionmodules.denoiser.DiscreteDenoiserWithControl",
                         "params": {"num_idx": 1000, "weighting_config": {"target": "sgm.modules.diffusionmodules.denoiser_weighting.EpsWeighting"},
                                    "scaling_config": {"target": "sgm.modules.diffusionmodules.denoiser_scaling.EpsScaling"},
                                    "discretization_config": disc}},
        first_stage_config={"target": "sgm.models.autoencoder.AutoencoderKLInferenceWrapper",
                            "params": {"embed_dim": 4, "ddconfig": vcfg, "lossconfig": {"target": "torch.nn.Identity"}}},
        sampler_config=sampler, ae_dtype="bf16", diffusion_dtype=diffusion_dtype, scale_factor=0.13025, p_p=", masterpiece",
        n_p="blurry, lowres")
    with torch.device("cuda"):
        m = smodel.SUPIRModel(**cfg)
    m.model.load_state_dict(make_state_dict(json.loads(str(gu["shapes"])), seed=31))
    sd_vae = make_state_dict(json.loads(str(gv["shapes"])), seed=71)
    sd_vae.update({"denoise_encoder." + k[len("encoder."):]: v for k, v in sd_vae.items() if k.startswith("encoder.")})
    m.first_stage_model.load_state_dict(sd_vae)
    return m


@pytest.mark.parametrize("tiled", [False, True])
def test_engine_fp16_end_to_end(monkeypatch, tiled):
    """SUPIRModel(diffusion_dtype="fp16") through batchify_sample (3 steps; the tiled sampler stacks 9 windows of a 32^2
    latent 4 per network call): no warning, finite, and within 3e-2 of the bf16 run with the same seed and noise."""
    img = (randn((1, 3, 256, 256), 200) * 0.5).clamp(-1, 1).cuda()
    c = {"crossattn": randn((1, 77, 2048), 201).cuda(), "vector": randn((1, 2816), 202).cuda()}
    uc = {"crossattn": randn((1, 77, 2048), 203).cuda(), "vector": randn((1, 2816), 204).cuda()}
    outs = {}
    for dt in ("fp16", "bf16"):
        m = _engine(dt, tiled)
        assert m.model.compute_dtype == (torch.float16 if dt == "fp16" else torch.bfloat16)
        monkeypatch.setattr(torch, "randn_like", _SeededNoise(5000))
        with warnings.catch_warnings(record=True) as rec:
            warnings.simplefilter("always")
            outs[dt] = m.batchify_sample(img, num_steps=3, restoration_scale=4.0, s_churn=5, s_noise=1.01, cfg_scale=4.0, seed=1234,
                                         control_scale=0.9, use_linear_CFG=True, cfg_scale_start=1.0, c=c, uc=uc).float().cpu()
        if dt == "fp16":
            assert not [str(r.message) for r in rec], [str(r.message) for r in rec]
        del m
        torch.cuda.empty_cache()
    assert bool(torch.isfinite(outs["fp16"]).all())
    e = _rel(outs["fp16"], outs["bf16"])
    print(f"engine ({'tiled' if tiled else 'untiled'}) fp16 vs bf16: rel_fro={e:.4g}")
    assert e <= 3e-2


def test_sharded_fp16_bit_identical_to_single_gpu():
    """The two-GPU harness of test_gpu_multigpu.py in fp16: the unit-sharded tiled sampler, the CFG-branch-parallel untiled
    sampler and the sharded VAE equal the single-GPU run bit for bit on every rank (skips below 2 GPUs)."""
    import subprocess
    import sys
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 CUDA devices")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29534", os.path.join(root, "tools", "check_multigpu.py"), "--dtype", "fp16"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=root)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    res = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("{")][-1])
    print(res)
    assert res["dtype"] == "fp16" and res["finite"]
    assert res["sampler_sharded_equals_single"] and res["identical_on_all_ranks"] and res["untiled_branch_parallel_equals_single"]
