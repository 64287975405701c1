"""GPU parity of the tensor-core kernels AT THE SHAPES bench.py TIMES (the batch-98 denoiser call of BASELINE configs[2]:
49 windows x CFG pair, 128x128 latent windows), through the C ABI, against plain PyTorch fp32 maths on the same
bf16-rounded operands. The shape list is the GEMM-class launch list of that call (SURVEY.md §8a rows a8/a9): every
epilogue the networks use, every N tile the dispatcher can pick, bf16 and fp32 outputs.
Attention covers the two self-attention shapes of the step, ragged key counts and adversarial logits that move the
online-softmax row maximum (and so rescale O) in every key block.

Tolerance (bf16 storage, fp32 accumulation, vs fp32): |err| <= 2e-2 + 2e-2 |ref| per element for GEMM / conv outputs of
unit scale; attention: |err| <= 1.5e-2 |ref| + 4e-3 max|ref| and relative Frobenius error <= 5e-3.
Reference call sites: sgm/modules/attention.py:84-110,222-285; openaimodel.py:330-356; SUPIR_v0.py:91-113."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
M1, M2 = 98 * 32 * 32, 98 * 64 * 64      # token rows of the batch-98 call at the 1280- and 640-channel levels


def _ops():
    from supir_b200 import _native, ops
    return ops, _native


def _rand(shape, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(BF)


def _gelu(x):
    return 0.5 * x * (1.0 + torch.erf(x * (1.0 / math.sqrt(2.0))))


def _ref_gemm(a, w, bias, residual, act, chunk=32768):
    """fp32 reference with the reference's rounding points (autocast: bf16 Linear output, then activation / residual)."""
    outs = []
    wt = w.float().t().contiguous()
    for r0 in range(0, a.shape[0], chunk):
        acc = a[r0:r0 + chunk].float() @ wt
        if bias is not None:
            acc = acc + bias
        if act == 2:      # GEGLU on interleaved [16 value | 16 gate] column groups (the packed layout of nets.FeedForward)
            v = acc.view(acc.shape[0], -1, 2, 16)
            xv, gv = v[:, :, 0].to(BF).float(), v[:, :, 1].to(BF).float()
            acc = (xv * _gelu(gv).to(BF).float()).reshape(acc.shape[0], -1)
        elif act == 1:
            acc = F.silu(acc.to(BF).float())
        if residual is not None:
            acc = acc.to(BF).float() + residual[r0:r0 + chunk].float()
        outs.append(acc)
    return torch.cat(outs, 0)


def _check(got, ref, what, atol=2e-2, rtol=2e-2):
    err = (got.float() - ref).abs()
    bad = err > (atol + rtol * ref.abs())
    nbad = int(bad.sum())
    assert nbad == 0, f"{what}: {nbad} elements out of tolerance, max err {float(err.max()):.4g} (ref max {float(ref.abs().max()):.4g})"
    assert bool(torch.isfinite(got.float()).all()), what


# (M, N, K, act, bias, residual): the GEMM-class launches that carry the step
GEMM_SHAPES = [
    (M1, 10240, 1280, 2, True, False),    # FeedForward GEGLU proj, 1280-ch level (90 per call)
    (M1, 1280, 5120, 0, True, True),      # FeedForward out + residual
    (M1, 1280, 1280, 0, True, True),      # attention to_out / proj_in / proj_out (+ residual)
    (M1, 3840, 1280, 0, False, False),    # fused QKV projection
    (M2, 5120, 640, 2, True, False),      # GEGLU at the 640-ch level (short K, epilogue bound)
    (M2, 640, 640, 0, True, True),        # to_out at the 640-ch level
    (M2, 640, 2560, 0, True, True),       # FeedForward out, 640-ch level
    (M2, 1920, 640, 0, False, False),     # fused QKV, 640-ch level
    (98 * 77, 4096, 2048, 0, False, False),   # text K|V projection (a slice of the fused [sum 2C, 2048] matrix)
    (M2, 320, 2880, 1, True, False),      # SiLU epilogue (ZeroSFT mlp_shared as a GEMM shape)
]


@pytest.mark.parametrize("shape", GEMM_SHAPES, ids=lambda s: "M%d_N%d_K%d_act%d%s%s" % (s[0], s[1], s[2], s[3], "_b" if s[4] else "", "_r" if s[5] else ""))
def test_gemm_bench_shapes_all_tiles_and_pair_modes(shape):
    ops, native = _ops()
    M, N, K, act, with_bias, with_res = shape
    a = _rand((M, K), 11)
    w = _rand((N, K), 12, 1.0 / math.sqrt(K))
    bias = (_rand((N,), 13, 0.2).float()) if with_bias else None
    n_out = N // 2 if act == 2 else N
    res = _rand((M, n_out), 14) if with_res else None
    ref = _ref_gemm(a, w, bias, res, act)
    lib = native.load()
    try:
        for bn in (0, 64, 128, 160, 256):
            lib.supir_set_gemm_tile_n(bn)
            out = torch.full((M, n_out), float("nan"), dtype=BF, device="cuda")
            ops.gemm(a, w, out, bias=bias, residual=res, act=act)
            _check(out, ref, f"gemm {shape} tile_n={bn}")
        lib.supir_set_gemm_tile_n(0)
        if act != 2:
            out32 = torch.full((M, n_out), float("nan"), dtype=torch.float32, device="cuda")
            ops.gemm(a, w, out32, bias=bias, residual=res, act=act)
            _check(out32, ref, f"gemm {shape} fp32 out")
    finally:
        lib.supir_set_gemm_tile_n(0)


# (B, H, W, Cin, Cout, rowvec, residual, act): ResBlock convs of the batch-98 call at its three resolutions + ZeroSFT convs
CONV_SHAPES = [
    (98, 128, 128, 320, 320, True, False, 0),     # in_layers conv + timestep embedding (rowvec), 1.6 M pixels
    (98, 128, 128, 320, 320, False, True, 0),     # out_layers conv + skip
    (98, 64, 64, 640, 640, True, True, 0),
    (98, 32, 32, 1280, 1280, True, True, 0),
    (98, 32, 32, 2560, 1280, True, False, 0),     # output block after the skip concat
    (98, 64, 64, 320, 128, False, False, 1),      # ZeroSFT mlp_shared (SiLU)
    (98, 32, 32, 128, 5120, False, False, 0),     # ZeroSFT gamma|beta, 2560 + 2560 channels
]


@pytest.mark.parametrize("shape", CONV_SHAPES, ids=lambda s: "B%d_%dx%d_%dto%d%s%s_act%d" % (s[0], s[1], s[2], s[3], s[4], "_rv" if s[5] else "", "_r" if s[6] else "", s[7]))
def test_conv3x3_bench_shapes(shape):
    ops, native = _ops()
    B, H, W, Cin, Cout, with_rv, with_res, act = shape
    torch.backends.cudnn.allow_tf32 = False
    x = _rand((B * H * W, Cin), 21)
    w = _rand((Cout, Cin, 3, 3), 22, 1.0 / math.sqrt(9 * Cin))
    bias = _rand((Cout,), 23, 0.2).float()
    rv = _rand((B, Cout), 24, 0.5).float() if with_rv else None
    res = _rand((B * H * W, Cout), 25) if with_res else None
    wp = w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous()
    # fp32 reference in image chunks (the fp32 NCHW copies of 1.6 M x 320 activations are large)
    ref = torch.empty((B * H * W, Cout), dtype=torch.float32, device="cuda")
    wf = w.float()
    step = 14
    for b0 in range(0, B, step):
        nb = min(step, B - b0)
        xi = x[b0 * H * W:(b0 + nb) * H * W].float().view(nb, H, W, Cin).permute(0, 3, 1, 2)
        y = F.conv2d(xi, wf, bias, padding=1)
        if rv is not None:
            y = y + rv[b0:b0 + nb, :, None, None]
        y = y.permute(0, 2, 3, 1).reshape(nb * H * W, Cout)
        if act == 1:
            y = F.silu(y.to(BF).float())
        if res is not None:
            y = y.to(BF).float() + res[b0 * H * W:(b0 + nb) * H * W].float()
        ref[b0 * H * W:(b0 + nb) * H * W] = y
    lib = native.load()
    try:
        for bn in (0, 256, 160, 128, 64):
            lib.supir_set_gemm_tile_n(bn)
            out = torch.full((B * H * W, Cout), float("nan"), dtype=BF, device="cuda")
            ops.conv3x3(x, B, H, W, wp, out, bias=bias, rowvec=rv, residual=res, act=act)
            _check(out, ref, f"conv {shape} tile_n={bn}")
    finally:
        lib.supir_set_gemm_tile_n(0)


# ----------------------------------------------------------------------------------------------------------------------
# attention
# ----------------------------------------------------------------------------------------------------------------------
def _ref_attention(q, k, v, B, H, Lq, Lk, scale):
    """softmax(q k^T scale) v in fp32, batch element by batch element (sgm/modules/attention.py:273-277)."""
    C = H * 64
    out = torch.empty((B * Lq, C), dtype=torch.float32, device="cuda")
    for b in range(B):
        qb = q[b * Lq:(b + 1) * Lq].float().view(Lq, H, 64).transpose(0, 1)
        kb = k[b * Lk:(b + 1) * Lk].float().view(Lk, H, 64).transpose(0, 1)
        vb = v[b * Lk:(b + 1) * Lk].float().view(Lk, H, 64).transpose(0, 1)
        p = torch.softmax(qb @ kb.transpose(1, 2) * scale, dim=-1)
        out[b * Lq:(b + 1) * Lq] = (p @ vb).transpose(0, 1).reshape(Lq, C)
    return out


def _check_attention(got, ref, what):
    err = (got.float() - ref).abs()
    mx = float(ref.abs().max())
    bad = int((err > 1.5e-2 * ref.abs() + 4e-3 * mx).sum())
    fro = float((got.float() - ref).norm() / ref.norm())
    print(f"{what}: rel_fro={fro:.3g} max_err={float(err.max()):.3g} (ref max {mx:.3g})")
    assert bad == 0 and fro <= 5e-3, f"{what}: {bad} elements out of tolerance, rel_fro {fro:.3g}, max err {float(err.max()):.4g} (ref max {mx:.4g})"


ATT_SHAPES = [(98, 10, 4096, 4096), (98, 20, 1024, 1024), (98, 10, 4096, 77), (98, 20, 1024, 77),
              (3, 5, 1000, 500), (2, 10, 1300, 640), (4, 3, 333, 96), (3, 2, 260, 128), (2, 20, 1024, 1024)]


# softmax variants: (exponent pairs of 4 emulated on the FMA pipe, probability pairs of 4 packed to bf16 on the ALU pipe)
ATT_MODES = {"default": (-1, -1), "xu_pack": (0, 0), "half_alu_pack": (0, 2), "alu_pack": (0, 4), "exp_emulation": (2, 0)}


def _set_attention_mode(lib, mode):
    emu, pack = ATT_MODES[mode]
    lib.supir_set_attention_exp_emulation(emu)
    lib.supir_set_attention_alu_pack(pack)


@pytest.mark.parametrize("mode", list(ATT_MODES))
@pytest.mark.parametrize("shape", ATT_SHAPES, ids=lambda s: "B%d_H%d_Lq%d_Lk%d" % s)
def test_attention_bench_shapes(shape, mode):
    ops, native = _ops()
    B, H, Lq, Lk = shape
    if mode != "default" and B * H * Lq * Lk > 2e9:
        pytest.skip("the largest shapes run once, in the default mode")
    C = H * 64
    q, k, v = _rand((B * Lq, C), 31, 1.5), _rand((B * Lk, C), 32, 1.5), _rand((B * Lk, C), 33)
    ref = _ref_attention(q, k, v, B, H, Lq, Lk, 0.125)
    lib = native.load()
    try:
        _set_attention_mode(lib, mode)
        out = torch.full((B * Lq, C), float("nan"), dtype=BF, device="cuda")
        ops.attention(q, k, v, out, B, H, Lq, Lk)
        _check_attention(out, ref, f"attention {shape} {mode}")
    finally:
        _set_attention_mode(lib, "default")


@pytest.mark.parametrize("mode", ["default", "xu_pack", "exp_emulation"])
@pytest.mark.parametrize("Lk", [1024, 4096, 640])
def test_attention_adversarial_logits_force_rescale(Lk, mode):
    """Key block j is aligned with the queries with a gain that grows with j, so the row maximum rises by ~9 log2 units
    (> the lazy-rescale threshold of 8) in EVERY 128-key block for the even query rows, while the odd rows keep their first
    maximum (both branches inside one warp); a few rows are all-equal (q = 0 -> uniform average of V)."""
    ops, native = _ops()
    B, H, Lq = 2, 10, 512
    C = H * 64
    g = torch.Generator(device="cuda").manual_seed(41)
    q = torch.randn((B, Lq, H, 64), generator=g, device="cuda")
    qdir = q / q.norm(dim=-1, keepdim=True)
    q = qdir * 8.0
    k = torch.randn((B, Lk, H, 64), generator=g, device="cuda") * 0.3
    # gain per key block: logits q.k*scale rise by 6.3 (natural units) = 9.1 log2 units per block along direction u
    u = qdir[:, 0::2].mean(dim=1, keepdim=True)
    u = u / u.norm(dim=-1, keepdim=True)
    q[:, 0::2] = u * 8.0 + 0.05 * q[:, 0::2]
    blocks = (torch.arange(Lk, device="cuda") // 128).float().view(1, Lk, 1, 1)
    k = k + u * (blocks * 6.3 / (8.0 * 0.125))
    q[:, 5] = 0.0
    q[:, 130] = 0.0
    v = torch.randn((B, Lk, H, 64), generator=g, device="cuda")
    qb, kb, vb = (t.reshape(B * t.shape[1], C).to(BF).contiguous() for t in (q, k, v))
    ref = _ref_attention(qb, kb, vb, B, H, Lq, Lk, 0.125)
    lib = native.load()
    try:
        _set_attention_mode(lib, mode)
        out = torch.full((B * Lq, C), float("nan"), dtype=BF, device="cuda")
        ops.attention(qb, kb, vb, out, B, H, Lq, Lk)
        _check_attention(out, ref, f"adversarial attention Lk={Lk} {mode}")
        # descending gain: the maximum sits in the first block and later blocks underflow towards zero probability
        kd = (k - u * (blocks * 6.3 / (8.0 * 0.125)) * 2).reshape(B * Lk, C).to(BF).contiguous()
        ref_d = _ref_attention(qb, kd, vb, B, H, Lq, Lk, 0.125)
        ops.attention(qb, kd, vb, out, B, H, Lq, Lk)
        _check_attention(out, ref_d, f"descending-logit attention Lk={Lk} {mode}")
    finally:
        _set_attention_mode(lib, "default")


@pytest.mark.parametrize("B,L,D", [(1, 18496, 512), (1, 22500, 512), (2, 300, 512), (1, 128, 512), (2, 777, 256), (3, 200, 128), (1, 4096, 128)])
def test_vae_single_head_attention(B, L, D):
    """The VAE mid-block attention (model.py:187-189; tilevae.py:292-336) at the token counts of the bench's padded tiles
    (136^2 = 18 496 for a 1088-px encoder tile, 150^2 = 22 500 for a 150-latent decoder tile) and ragged small cases."""
    ops, native = _ops()
    q, k, v = _rand((B * L, D), 51, 1.0), _rand((B * L, D), 52, 1.0), _rand((B * L, D), 53)
    scale = D ** -0.5
    ref = torch.empty((B * L, D), dtype=torch.float32, device="cuda")
    for b in range(B):
        sl = slice(b * L, (b + 1) * L)
        for r0 in range(0, L, 4096):
            p = torch.softmax(q[sl][r0:r0 + 4096].float() @ k[sl].float().t() * scale, dim=-1)
            ref[b * L + r0:b * L + min(r0 + 4096, L)] = p @ v[sl].float()
    out = torch.full((B * L, D), float("nan"), dtype=BF, device="cuda")
    ops.attention_1head(q, k, v, out, B, L)
    _check_attention(out, ref, f"single-head attention B={B} L={L} D={D}")
    # operands as column slices of a fused [L, 3D] projection (how the VAE calls it)
    qkv = torch.cat([q, k, v], 1).contiguous()
    out2 = torch.full((B * L, D), float("nan"), dtype=BF, device="cuda")
    ops.attention_1head(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:], out2, B, L)
    assert torch.equal(out, out2)
