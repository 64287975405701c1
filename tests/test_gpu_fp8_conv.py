"""GPU tests of the FP8 convs option (supir_conv3x3_fp8, supir_groupnorm_apply_quant and ControlWrapper.fp8_convs on top of
dtype=torch.float8_e4m3fn).

GroupNorm-quant is checked against torch's quantization of an fp32 GroupNorm + SiLU: scales to fp32 rounding, codes within half an
e4m3 step, as for LayerNorm-quant; the scale is per image. The convolution is checked against an fp64 convolution of the
DEQUANTIZED operands, with the bf16 rounding of the output (and of the epilogue's rounding points) and an absolute term for the
tensor cores' accumulation over K = 9 Cin. Networks: the depth-1 full-width networks against the fp32 oracle with and without
fake quantization at exactly the FP8 points, graph replay, mode switching, row independence, sharding and the engine.
"""
import json
import os
import warnings

import pytest
import torch
import torch.nn.functional as F

from test_gpu_fp8 import FP8_LAYERS, _engine, _depth1, _fake_quant, _inputs, _Out, _oracle, _rand, _rel, _SeededNoise
from weights import randn

pytestmark = pytest.mark.gpu
BF, FP8 = torch.bfloat16, torch.float8_e4m3fn


def _ops():
    from supir_b200 import _native, nets, ops
    return ops, nets, _native.load()


def _image_quant(x, B):
    """Per-image codes and scales of fp32 NHWC rows x [B*HW, C] (the contract's formula over each image's HW*C values)."""
    from supir_b200 import ops
    xi = x.reshape(B, -1)
    s, inv = ops.e4m3_row_scales(xi)
    return (xi * inv[:, None]).to(FP8).view(x.shape), s


# ---------------------------------------------------------------------------------------------------------------------
# GroupNorm + SiLU -> e4m3
# ---------------------------------------------------------------------------------------------------------------------
def _gn_quant(x, B, HW, gamma, beta):
    ops, _, _ = _ops()
    C = x.shape[1]
    sums = torch.zeros(ops.groupnorm_ws_size(B, HW, C), dtype=torch.float64, device="cuda")
    ops.groupnorm_stats(x, B, HW, sums)
    q, s = _Out(B * HW, C, FP8), torch.full((B,), float("nan"), device="cuda")
    amax = torch.full((B,), -1, dtype=torch.int32, device="cuda")              # stale contents: the call resets it
    ops.groupnorm_apply_quant(x, B, HW, q.view, s, amax, gamma, beta, 1e-5, True, sums)
    return q.done(), s


@pytest.mark.parametrize("B,HW,C", [(1, 64, 320), (2, 1024, 640), (3, 300, 960), (2, 4096, 1280), (1, 100, 2560), (34, 256, 320)])
def test_groupnorm_apply_quant_against_torch(B, HW, C):
    x = _rand((B, HW, C), C + HW) * 2 + 0.5
    x = (x * torch.exp(2 * _rand((B, 1, 1), 7))).reshape(B * HW, C).to(BF)            # very different image scales
    gamma, beta = 1 + 0.2 * _rand((C,), 2), 0.1 * _rand((C,), 3)
    got, s = _gn_quant(x, B, HW, gamma, beta)
    xt = x.float().view(B, HW, C).permute(0, 2, 1)
    y = F.silu(F.group_norm(xt, 32, gamma, beta, 1e-5)).permute(0, 2, 1).reshape(B * HW, C)
    rq, rs = _image_quant(y, B)
    assert bool(torch.isfinite(s).all())
    assert torch.allclose(s, rs, rtol=1e-5, atol=0), (s, rs)
    si = s.repeat_interleave(HW)[:, None]
    deq = got.float() * si
    # half an e4m3 step (2^-4 relative for normals, 2^-10 * scale absolute for subnormals) plus fp32 GroupNorm noise
    amax = (rs * 448).repeat_interleave(HW)[:, None]
    tol = (2.0 ** -4) * y.abs() + (2.0 ** -9) * si + 1e-5 * amax
    assert bool(((deq - y).abs() <= tol).all()), float(((deq - y).abs() - tol).max())
    same = float((got.view(torch.uint8) == rq.view(torch.uint8)).float().mean())
    assert same > 0.99, same


def test_groupnorm_apply_quant_scale_is_per_image():
    """An image alone gives the codes and the scale it has inside a batch, bit for bit."""
    B, HW, C = 3, 576, 640
    x = (_rand((B, HW, C), 21) * torch.tensor([0.01, 1.0, 50.0], device="cuda")[:, None, None]).reshape(B * HW, C).to(BF)
    gamma, beta = 1 + 0.2 * _rand((C,), 22), 0.1 * _rand((C,), 23)
    full, s = _gn_quant(x, B, HW, gamma, beta)
    for i in range(B):
        one, s1 = _gn_quant(x[i * HW:(i + 1) * HW].contiguous(), 1, HW, gamma, beta)
        assert torch.equal(one.view(torch.uint8), full[i * HW:(i + 1) * HW].view(torch.uint8)) and float(s1[0]) == float(s[i]), i


# ---------------------------------------------------------------------------------------------------------------------
# conv3x3_fp8
# ---------------------------------------------------------------------------------------------------------------------
def _bf(x):
    return x.to(BF).to(x.dtype)


def _conv_case(B, H, W, Cin, Cout, epi, bn, img_scales=None, seed=0):
    ops, nets, lib = _ops()
    M = B * H * W
    x = _rand((B, H * W, Cin), 31 + seed + Cin)
    if img_scales is not None:
        x = x * torch.tensor(img_scales, device="cuda")[:, None, None]
    x = x.reshape(M, Cin)
    xq, xs = _image_quant(x, B)
    w = _rand((Cout, Cin, 3, 3), 32 + seed + Cout, (9 * Cin) ** -0.5)
    wq, ws = ops.quantize_weight(nets.pack_conv3x3(w))
    to_nchw = lambda t: t.view(B, H, W, -1).permute(0, 3, 1, 2)                 # noqa: E731
    xd = xq.double() * xs.double().repeat_interleave(H * W)[:, None]
    wd = (wq.double() * ws.double()[:, None]).view(Cout, 3, 3, Cin).permute(0, 3, 1, 2)
    acc = F.conv2d(to_nchw(xd), wd, padding=1).permute(0, 2, 3, 1).reshape(M, Cout)
    absum = F.conv2d(to_nchw(xd.abs()), wd.abs(), padding=1).permute(0, 2, 3, 1).reshape(M, Cout)
    bias = _bf(_rand((Cout,), 33, 0.5))
    rv_full = _rand((B, Cout + 64), 34)
    rv = rv_full[:, 32:32 + Cout]                                                # a per-image vector with rowvec_ld > Cout
    res = _rand((M, Cout), 35).to(BF)
    pre = acc
    kw = {}
    if epi == "bias_rowvec":
        pre = acc + bias.double() + rv.double().repeat_interleave(H * W, 0)
        kw, ref = dict(bias=bias, rowvec=rv), pre
    elif epi == "residual":
        pre = acc + bias.double()
        kw, ref = dict(bias=bias, residual=res), _bf(pre) + res.double()
    elif epi == "silu":
        pre = acc + bias.double()
        kw, ref = dict(bias=bias, act=1), F.silu(_bf(pre))
    else:
        ref = acc
    o = _Out(M, Cout, BF)
    lib.supir_set_gemm_tile_n(bn)
    try:
        ops.conv3x3_fp8(xq, xs, B, H, W, wq, ws, o.view, **kw)
    finally:
        lib.supir_set_gemm_tile_n(0)
    got = o.done().double()
    assert bool(torch.isfinite(got).all()), f"{int((~torch.isfinite(got)).sum())} unwritten outputs"
    # bf16 rounding of the result (2^-7 relative) and of the rounding point before the residual / SiLU, plus the tensor cores'
    # e4m3 accumulation over K = 9 Cin: 2^-9 of the sum of |products| of the element (it only shows where the sum cancels)
    u, c = 2.0 ** -7, 2.0 ** -9
    tol = u * ref.abs() + c * absum
    if epi in ("residual", "silu"):
        tol = tol + 1.1 * u * pre.abs()
    err = (got - ref).abs()
    nbad = int((err > tol).sum())
    worst = float((err / tol).max())
    assert nbad == 0, (f"B={B} H={H} W={W} Cin={Cin} Cout={Cout} {epi} bn={bn}: {nbad} out of tolerance, max err "
                       f"{float(err.max()):.3g}, err/tol {worst:.3g}")
    return worst


@pytest.mark.parametrize("bn", [0, 64, 128, 160, 256])
@pytest.mark.parametrize("epi", ["none", "bias_rowvec", "residual", "silu"])
def test_conv3x3_fp8_epilogues_and_widths(epi, bn):
    """Every forced width (64 / 128: ping-pong, 160 / 256: cooperative) with H and W tails and a partial last n-tile."""
    _conv_case(2, 13, 21, 320, 640, epi, bn)


@pytest.mark.parametrize("Cin,Cout", [(320, 320), (640, 640), (960, 640), (1280, 1280), (2560, 1280)])
@pytest.mark.parametrize("H,W", [(16, 16), (9, 40)])
def test_conv3x3_fp8_channel_counts(Cin, Cout, H, W):
    """The ResBlock conv rows of the step: Cin 320 and 960 are not multiples of the 128-channel k-block (zero fill past Cin)."""
    _conv_case(2, H, W, Cin, Cout, "bias_rowvec", 0)
    _conv_case(1, H, W, Cout, Cout, "residual", 0)


def test_conv3x3_fp8_per_image_scales():
    """B = 3 with image magnitudes 1e-3 / 1 / 1e3: each image's result is checked against its own scale."""
    for bn in (0, 128, 256):
        _conv_case(3, 12, 20, 640, 640, "none", bn, img_scales=[1e-3, 1.0, 1e3], seed=5)


# ---------------------------------------------------------------------------------------------------------------------
# networks
# ---------------------------------------------------------------------------------------------------------------------
def _wrapper(cfg, sd, dtype, fp8_convs):
    from supir_b200 import nets, wrappers
    with torch.device("cuda"):
        unet = nets.LightGLVUNet(mode="XL-base", project_type="ZeroSFT", project_channel_scale=2, **cfg)
        ctrl = nets.GLVControl(input_upscale=1, **cfg)
    w = wrappers.ControlWrapper(unet, dtype=dtype)
    w.fp8_convs = fp8_convs
    w.load_control_model(ctrl)
    w.load_state_dict(sd, strict=True)
    return w


FP8_CONVS = (".in_layers.2", ".out_layers.3")


def _fake_quant_image(x):
    """Per-image e4m3 fake quantization of an NCHW tensor (one scale over C*H*W)."""
    from supir_b200 import ops
    x2 = x.reshape(x.shape[0], -1).float()
    s, inv = ops.e4m3_row_scales(x2)
    return ((x2 * inv[:, None]).to(FP8).float() * s[:, None]).reshape(x.shape)


# measured on an H100 80GB HBM3 at 700 W (see DESIGN.md section 7): 0.0325 and 0.0377, with margin
FAKE_ORACLE_BOUND = 0.045
PLAIN_ORACLE_BOUND = 0.055


def test_network_fp8_convs_vs_oracle_with_and_without_fake_quantization(monkeypatch):
    """(a) against the oracle with e4m3 fake quantization at exactly the FP8 points: the transformer blocks' linears (per row) and
    the ResBlocks' 3x3 convolutions (weights per output channel of the bf16 matrix, inputs per image); (b) against the plain
    oracle; (a) below (b), both pinned."""
    from oracle import unet as ounet
    cfg, sd = _depth1()
    x, t, cond = _inputs(2)
    cc = {k: v.cuda() for k, v in cond.items()}
    w = _wrapper(cfg, sd, FP8, True)
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        out = w(x.cuda(), t.cuda(), cc, control_scale=0.8).cpu()
    assert bool(torch.isfinite(out).all())
    plain = _oracle(sd, x, t, cond, 0.8)
    lin0, conv0 = ounet._lin, ounet._conv

    def lin(sdd, p, xx):
        if ".transformer_blocks." in p and p.endswith(FP8_LAYERS):
            wq = _fake_quant(sdd[p + ".weight"].to(BF).float())
            return F.linear(_fake_quant(xx), wq, sdd.get(p + ".bias"))
        return lin0(sdd, p, xx)

    def conv(sdd, p, xx, stride=1, padding=1):
        if p.endswith(FP8_CONVS):
            wt = sdd[p + ".weight"].to(BF).float()
            wq = _fake_quant(wt.reshape(wt.shape[0], -1)).reshape(wt.shape)
            return F.conv2d(_fake_quant_image(xx), wq, sdd.get(p + ".bias"), stride=stride, padding=padding)
        return conv0(sdd, p, xx, stride=stride, padding=padding)

    monkeypatch.setattr(ounet, "_lin", lin)
    monkeypatch.setattr(ounet, "_conv", conv)
    fake = _oracle(sd, x, t, cond, 0.8)
    ea, eb = _rel(out, fake), _rel(out, plain)
    print(f"depth-1 FP8 linears + convs networks: vs fake-quantized oracle {ea:.4g}, vs plain oracle {eb:.4g} "
          f"(|fake - plain| / |plain| = {_rel(fake, plain):.4g})")
    assert ea <= FAKE_ORACLE_BOUND
    assert eb <= PLAIN_ORACLE_BOUND
    assert ea < eb


def test_graph_replay_and_mode_switch():
    """bf16 -> fp8 -> fp8 + convs -> fp8 -> fp8 + convs: each mode gives back its earlier output bit for bit; replay = eager."""
    cfg, sd = _depth1()
    x, t, cond = _inputs(2)
    args = (x.cuda(), t.cuda(), {k: v.cuda() for k, v in cond.items()})
    w = _wrapper(cfg, sd, BF, False)
    b1 = w(*args, control_scale=0.8).clone()
    w.dtype = FP8
    f1 = w(*args, control_scale=0.8).clone()
    w.fp8_convs = True
    assert not w._packed and not w._plans
    c1 = w(*args, control_scale=0.8).clone()
    plan = next(iter(w._plans.values()))
    assert plan.graph is not None
    plan.out.fill_(float("nan"))
    plan._run()
    torch.cuda.synchronize()
    eager = plan.out.clone()
    c2 = w(*args, control_scale=0.8).clone()
    assert bool(torch.isfinite(eager).all()) and torch.equal(eager, c1) and torch.equal(eager, c2)
    assert not torch.equal(c1, f1) and not torch.equal(f1, b1)
    w.fp8_convs = False
    assert torch.equal(w(*args, control_scale=0.8), f1)
    w.fp8_convs = True
    assert torch.equal(w(*args, control_scale=0.8), c1)
    w.fp8_convs = False
    w.dtype = BF
    assert torch.equal(w(*args, control_scale=0.8), b1)


def test_rows_independent():
    """A batch equals its rows computed separately, bit for bit (per-image activation scales)."""
    cfg, sd = _depth1()
    x, t, cond = _inputs(4, side=8)
    w = _wrapper(cfg, sd, FP8, True)
    full = w(x.cuda(), t.cuda(), {k: v.cuda() for k, v in cond.items()}, control_scale=1.0).clone()
    for i in (0, 3):
        one = w(x[i:i + 1].cuda(), t[i:i + 1].cuda(), {k: v[i:i + 1].cuda() for k, v in cond.items()}, control_scale=1.0)
        assert torch.equal(one[0], full[i]), i


def test_sharded_fp8_convs_bit_identical_to_single_gpu():
    import subprocess
    import sys
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 CUDA devices")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29537", os.path.join(root, "tools", "check_multigpu.py"), "--fp8-convs"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=root)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    res = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("{")][-1])
    assert res["dtype"] == "fp8" and res["fp8_convs"] and res["finite"] and res["sampler_sharded_equals_single"]
    assert res["identical_on_all_ranks"]


# measured on an H100 80GB HBM3 at 700 W (see DESIGN.md section 7): 0.0486 untiled, 0.0518 tiled, with margin
ENGINE_BOUND = 0.08


@pytest.mark.parametrize("tiled", [False, True])
def test_engine_fp8_convs_end_to_end(monkeypatch, tiled):
    img = (randn((1, 3, 256, 256), 200) * 0.5).clamp(-1, 1).cuda()
    c = {"crossattn": randn((1, 77, 2048), 201).cuda(), "vector": randn((1, 2816), 202).cuda()}
    uc = {"crossattn": randn((1, 77, 2048), 203).cuda(), "vector": randn((1, 2816), 204).cuda()}
    outs = {}
    for dt in ("fp8", "bf16"):
        m = _engine(dt, tiled)
        if dt == "fp8":
            m.model.fp8_convs = True                # the drop-in route after --diff_dtype fp8
        monkeypatch.setattr(torch, "randn_like", _SeededNoise(5000))
        with warnings.catch_warnings(record=True) as rec:
            warnings.simplefilter("always")
            outs[dt] = m.batchify_sample(img, num_steps=3, restoration_scale=4.0, s_churn=5, s_noise=1.01, cfg_scale=4.0, seed=1234,
                                         control_scale=0.9, use_linear_CFG=True, cfg_scale_start=1.0, c=c, uc=uc).float().cpu()
        if dt == "fp8":
            assert not [str(r.message) for r in rec], [str(r.message) for r in rec]
            assert m.model.diffusion_model._fp8_linears and m.model.diffusion_model._fp8_convs
        del m
        torch.cuda.empty_cache()
    assert bool(torch.isfinite(outs["fp8"]).all())
    e = _rel(outs["fp8"], outs["bf16"])
    print(f"engine ({'tiled' if tiled else 'untiled'}) fp8 linears + convs vs bf16: rel_fro={e:.4g}")
    assert e <= ENGINE_BOUND
