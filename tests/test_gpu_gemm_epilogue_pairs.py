"""GPU tests of the GEMM epilogue's column-operand loads: each column operand (bias, folded LayerNorm column sums, per-batch
vector, e4m3 weight scales) is read once per fragment as 64-bit pairs when the tile lies inside N and the operand is 8-byte
aligned, and as 32-bit loads otherwise (ragged last n-tile, odd N, operands at an odd float offset).

Every case runs at each tile width and must give bit-identical outputs across the widths (the arithmetic and its rounding
points do not depend on the width), and the 64-bit path must agree bit for bit with the same operands at an odd float
offset (32-bit path). The outputs must also match plain PyTorch fp32 maths on the same 16-bit operands. The per-batch
vector cases put a batch boundary between the two rows a thread holds."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
WIDTHS = (64, 128, 160, 256)
DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}


def _ops():
    from supir_b200 import _native, ops
    return ops, _native.load()


def _randf(shape, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(shape, generator=g, device="cuda") * scale


def _misaligned(t):
    """a copy of fp32 vector or matrix `t` at an odd float offset (4-byte, not 8-byte aligned)"""
    buf = torch.empty(t.numel() + 1, dtype=torch.float32, device="cuda")
    v = buf[1:].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 8 == 4
    return v


def _at_widths(lib, run):
    outs = []
    for bn in WIDTHS:
        lib.supir_set_gemm_tile_n(bn)
        try:
            outs.append(run())
        finally:
            lib.supir_set_gemm_tile_n(0)
    torch.cuda.synchronize()
    return outs


def _same(outs, what):
    for bn, o in zip(WIDTHS[1:], outs[1:]):
        nd = int((o.view(torch.int16) != outs[0].view(torch.int16)).sum())
        assert nd == 0, f"{what}: width {bn} differs from width {WIDTHS[0]} in {nd} elements"


def _close(out, ref, what):
    err = (out.float() - ref).abs()
    bad = err > 2e-2 + 2e-2 * ref.abs()
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} elements off fp32 maths, max error {float(err.max()):.4g}"


# (M, N, K): a ragged last m-tile and n-tile, odd N, one tile, many tiles per CTA
SHAPES = [(300, 640, 256), (1000, 1280, 320), (129, 161, 128), (77, 96, 64), (4099, 1920, 192)]


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("epi", ["bias+res", "ln+bias", "rowvec+silu"])
def test_epilogue_column_pairs(dt, M, N, K, epi):
    ops, lib = _ops()
    dtype = DTYPES[dt]
    a = _randf((M, K), 1).to(dtype)
    w = (_randf((N, K), 2) / K ** 0.5).to(dtype)
    bias = _randf((N,), 3)
    res = _randf((M, N), 4).to(dtype) if "res" in epi else None
    rpb = 37                                      # a batch boundary between a thread's rows r and r + 8
    nb = (M + rpb - 1) // rpb
    rowvec = _randf((nb, N), 5) if "rowvec" in epi else None
    ln = (torch.stack([_randf((M,), 6).abs() + 0.5, _randf((M,), 7)], 1).contiguous(), _randf((N,), 8)) if "ln" in epi else None
    act = 1 if "silu" in epi else 0

    def run(bias=bias, rowvec=rowvec, ln=ln):
        out = torch.empty(M, N, dtype=dtype, device="cuda")
        return ops.gemm(a, w, out, bias=bias, rowvec=rowvec, rows_per_batch=rpb if rowvec is not None else 0, residual=res,
                        act=act, ln=ln)

    outs = _at_widths(lib, run)
    _same(outs, f"{epi} {M}x{N}x{K} {dt}")
    odd = _at_widths(lib, lambda: run(bias=_misaligned(bias), rowvec=None if rowvec is None else _misaligned(rowvec),
                                      ln=None if ln is None else (ln[0], _misaligned(ln[1]))))
    for bn, o, e in zip(WIDTHS, outs, odd):
        assert bool((o.view(torch.int16) == e.view(torch.int16)).all()), f"{epi} {M}x{N}x{K} {dt}: width {bn}: 64-bit and 32-bit loads differ"

    acc = a.float() @ w.float().t()
    if ln is not None:
        acc = acc * ln[0][:, :1] - ln[0][:, 1:] * ln[1][None, :]
    acc = acc + bias
    if rowvec is not None:
        acc = acc + rowvec[torch.arange(M, device="cuda") // rpb]
    if act == 1:
        acc = F.silu(acc.to(dtype).float())
    if res is not None:
        acc = acc.to(dtype).float() + res.float()
    _close(outs[0], acc, f"{epi} {M}x{N}x{K} {dt}")


@pytest.mark.parametrize("M,N,K", [(300, 1280, 256), (129, 256, 128), (1000, 640, 192)])
def test_geglu_column_pairs(M, N, K):
    ops, lib = _ops()
    a = _randf((M, K), 11).to(torch.bfloat16)
    w = (_randf((N, K), 12) / K ** 0.5).to(torch.bfloat16)
    bias = _randf((N,), 13)
    res = _randf((M, N // 2), 14).to(torch.bfloat16)

    def run(bias=bias):
        out = torch.empty(M, N // 2, dtype=torch.bfloat16, device="cuda")
        return ops.gemm(a, w, out, bias=bias, residual=res, act=2)

    outs = _at_widths(lib, run)
    _same(outs, f"geglu {M}x{N}x{K}")
    odd = _at_widths(lib, lambda: run(bias=_misaligned(bias)))
    for bn, o, e in zip(WIDTHS, outs, odd):
        assert bool((o.view(torch.int16) == e.view(torch.int16)).all()), f"geglu {M}x{N}x{K}: width {bn}: 64-bit and 32-bit loads differ"
    acc = (a.float() @ w.float().t() + bias).view(M, N // 32, 2, 16)
    x, g = acc[:, :, 0].reshape(M, N // 2), acc[:, :, 1].reshape(M, N // 2)
    bf = lambda t: t.to(torch.bfloat16).float()  # noqa: E731
    ref = bf(bf(x) * bf(F.gelu(bf(g)))) + res.float()
    _close(outs[0], ref, f"geglu {M}x{N}x{K}")


def _check(lib, run, run_odd, ref, what):
    """`run` at every width: bit-identical across widths and to `run_odd` (32-bit loads) at each width, and close to `ref`"""
    outs = _at_widths(lib, run)
    _same(outs, what)
    odd = _at_widths(lib, run_odd)
    for bn, o, e in zip(WIDTHS, outs, odd):
        assert bool((o.view(torch.int16) == e.view(torch.int16)).all()), f"{what}: width {bn}: 64-bit and 32-bit loads differ"
    _close(outs[0], ref, what)


def _nchw(x, B, H, W):
    return x.float().view(B, H, W, -1).permute(0, 3, 1, 2)


def _nhwc(y):
    return y.permute(0, 2, 3, 1).reshape(-1, y.shape[1])


# patches that run past the image (rows whose partner row is outside it), a ragged last n-tile (Cout 200)
@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("B,H,W,Cout", [(3, 13, 21, 200), (2, 16, 16, 320)])
def test_conv3x3_column_pairs(dt, B, H, W, Cout):
    ops, lib = _ops()
    dtype, Cin = DTYPES[dt], 64
    x = _randf((B * H * W, Cin), 21).to(dtype)
    w = _randf((Cout, Cin, 3, 3), 22, (9 * Cin) ** -0.5).to(dtype)
    wp = w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous()
    bias, rv, res = _randf((Cout,), 23), _randf((B, Cout), 24), _randf((B * H * W, Cout), 25).to(dtype)

    def run(bias=bias, rv=rv):
        out = torch.empty(B * H * W, Cout, dtype=dtype, device="cuda")
        return ops.conv3x3(x, B, H, W, wp, out, bias=bias, rowvec=rv, residual=res, act=1)

    y = F.conv2d(_nchw(x, B, H, W), w.float(), bias, padding=1) + rv[:, :, None, None]
    ref = F.silu(_nhwc(y).to(dtype).float()).to(dtype).float() + res.float()
    _check(lib, run, lambda: run(bias=_misaligned(bias), rv=_misaligned(rv)), ref, f"conv3x3 {B}x{H}x{W}->{Cout} {dt}")


@pytest.mark.parametrize("pad_lo", [1, 0])
def test_conv_stride2_column_pairs(pad_lo):
    ops, lib = _ops()
    B, H, W, Cin, Cout = 2, 30, 22, 64, 200
    x = _randf((B * H * W, Cin), 31).to(torch.bfloat16)
    w = _randf((Cout, Cin, 3, 3), 32, (9 * Cin) ** -0.5).to(torch.bfloat16)
    wp = w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous()
    bias = _randf((Cout,), 33)
    xi = _nchw(x, B, H, W)
    y = F.conv2d(xi, w.float(), bias, stride=2, padding=1) if pad_lo else F.conv2d(F.pad(xi, (0, 1, 0, 1)), w.float(), bias, stride=2)

    def run(bias=bias):
        out = torch.empty(B * y.shape[2] * y.shape[3], Cout, dtype=torch.bfloat16, device="cuda")
        return ops.conv3x3_stride2(x, B, H, W, wp, out, pad_lo, bias=bias)

    _check(lib, run, lambda: run(bias=_misaligned(bias)), _nhwc(y), f"conv stride 2 pad_lo={pad_lo}")


def test_upsample2x_column_pairs():
    """four sub-pixel convolutions, each storing every second pixel of every second output row"""
    ops, lib = _ops()
    B, H, W, Cin, Cout = 2, 11, 17, 64, 200
    x = _randf((B * H * W, Cin), 41).to(torch.bfloat16)
    w = _randf((Cout, Cin, 3, 3), 42, (9 * Cin) ** -0.5)
    bias = _randf((Cout,), 43)
    wfold = ops.fold_upsample_weights(w, torch.bfloat16)
    y = F.conv2d(F.interpolate(_nchw(x, B, H, W), scale_factor=2, mode="nearest"), w.to(torch.bfloat16).float(), bias, padding=1)

    def run(bias=bias):
        out = torch.empty(B * 4 * H * W, Cout, dtype=torch.bfloat16, device="cuda")
        return ops.upsample2x_conv3x3(x, B, H, W, wfold, out, bias=bias)

    _check(lib, run, lambda: run(bias=_misaligned(bias)), _nhwc(y), "upsample2x conv")


def _e4m3(shape, seed):
    return (_randf(shape, seed) * 64).clamp(-448, 448).to(torch.float8_e4m3fn)


@pytest.mark.parametrize("M,N,K,act", [(300, 1280, 256, 0), (129, 200, 128, 0), (1000, 640, 192, 2)])
def test_fp8_gemm_column_pairs(M, N, K, act):
    """e4m3 with per-row scales of both operands: the accumulator times a_scale[m] * w_scale[n] comes first"""
    ops, lib = _ops()
    a_q, w_q = _e4m3((M, K), 51), _e4m3((N, K), 52)
    # outputs of order 1: the GEGLU's bf16 rounding points then keep the fp32 reference within the tolerance
    a_s, w_s = _randf((M,), 53).abs() * 1e-3 + 1e-4, _randf((N,), 54).abs() * 1e-3 + 1e-4
    bias = _randf((N,), 55)
    n_out = N // 2 if act == 2 else N
    res = _randf((M, n_out), 56).to(torch.bfloat16)

    def run(w_s=w_s, bias=bias):
        out = torch.empty(M, n_out, dtype=torch.bfloat16, device="cuda")
        return ops.gemm_fp8(a_q, a_s, w_q, w_s, out, bias=bias, residual=res, act=act)

    acc = a_s[:, None] * w_s[None, :] * (a_q.float() @ w_q.float().t()) + bias
    bf = lambda t: t.to(torch.bfloat16).float()  # noqa: E731
    if act == 2:
        acc = acc.view(M, N // 32, 2, 16)
        xv, g = acc[:, :, 0].reshape(M, n_out), acc[:, :, 1].reshape(M, n_out)
        ref = bf(bf(xv) * bf(F.gelu(bf(g)))) + res.float()
    else:
        ref = bf(acc) + res.float()
    _check(lib, run, lambda: run(w_s=_misaligned(w_s), bias=_misaligned(bias)), ref, f"fp8 gemm {M}x{N}x{K} act {act}")


def test_fp8_conv_column_pairs():
    """e4m3 convolution: one activation scale per image, patches past the image, ragged last n-tile"""
    ops, lib = _ops()
    B, H, W, Cin, Cout = 3, 13, 21, 64, 200
    x_q, w_q = _e4m3((B * H * W, Cin), 61), _e4m3((Cout, 9 * Cin), 62)
    x_s, w_s = _randf((B,), 63).abs() * 1e-2 + 1e-3, _randf((Cout,), 64).abs() * 1e-3 + 1e-4
    bias, rv, res = _randf((Cout,), 65), _randf((B, Cout), 66), _randf((B * H * W, Cout), 67).to(torch.bfloat16)

    def run(w_s=w_s, bias=bias, rv=rv):
        out = torch.empty(B * H * W, Cout, dtype=torch.bfloat16, device="cuda")
        return ops.conv3x3_fp8(x_q, x_s, B, H, W, w_q, w_s, out, bias=bias, rowvec=rv, residual=res)

    w4 = w_q.float().view(Cout, 3, 3, Cin).permute(0, 3, 1, 2)
    y = F.conv2d(_nchw(x_q, B, H, W), w4, padding=1) * x_s[:, None, None, None] * w_s[None, :, None, None]
    y = y + bias[None, :, None, None] + rv[:, :, None, None]
    ref = _nhwc(y).to(torch.bfloat16).float() + res.float()
    _check(lib, run, lambda: run(w_s=_misaligned(w_s), bias=_misaligned(bias), rv=_misaligned(rv)), ref, "fp8 conv3x3")
