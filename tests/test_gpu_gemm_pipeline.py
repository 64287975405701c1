"""GPU tests of the wgmma GEMM / implicit-GEMM convolution kernel's persistent tile loop and epilogue, through the C ABI,
against plain PyTorch fp32 maths on the same bf16 operands (tolerance 2e-2 + 2e-2 |ref| per element, as in
test_gpu_bench_shapes.py).

Where test_gpu_bench_shapes.py covers the large shapes of the benchmark, this file covers the edges:
- tile counts per launch of 1, 2, SMs - 1, SMs + 1 and 2 SMs + 1, so the persistent CTAs get unequal numbers of tiles and
  some get none; at tile widths 64 and 128 (the ping-pong schedule) this gives the two consumer warpgroups of a CTA odd and
  even tile counts, one tile between them, or none, which is where the ordered hand-off between their mainloops must end
  without a dangling barrier arrival;
- M and N that are not multiples of the tile;
- every epilogue (bias, per-image vector with a batch boundary inside a tile, folded LayerNorm, SiLU, GEGLU, residual
  from a column slice, fp32 output) and every forced tile width;
- output into a column slice of a wider tensor, and at an odd leading dimension (the unaligned store path);
- ragged and stride-2 convolutions, the interleaved sub-pixel output of nearest-2x + conv3x3, conv + per-image vector +
  residual.
Outputs are written into NaN-filled buffers whose columns outside the written slice hold a sentinel value, so an
unwritten element fails the tolerance check and an element written outside the slice fails the sentinel check."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
WIDTHS = (0, 64, 128, 160, 256)
SENTINEL = 7.0


def _ops():
    from supir_b200 import _native, ops
    return ops, _native.load()


def _rand(shape, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(BF)


def _randf(shape, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(shape, generator=g, device="cuda") * scale


def _gelu(x):
    return 0.5 * x * (1.0 + torch.erf(x * (1.0 / math.sqrt(2.0))))


def _check(got, ref, what, atol=2e-2, rtol=2e-2):
    g = got.float()
    assert bool(torch.isfinite(g).all()), f"{what}: {int((~torch.isfinite(g)).sum())} non-finite (unwritten?) elements"
    err = (g - ref).abs()
    nbad = int((err > atol + rtol * ref.abs()).sum())
    assert nbad == 0, f"{what}: {nbad} elements out of tolerance, max err {float(err.max()):.4g}"


class _Slice:
    """A [rows, cols] output view at column offset `lo` of a wider buffer; the view starts NaN, the rest holds SENTINEL."""

    def __init__(self, rows, cols, lo=0, hi=0, dtype=BF):
        self.full = torch.full((rows, lo + cols + hi), SENTINEL, dtype=dtype, device="cuda")
        self.lo, self.cols = lo, cols
        self.view = self.full[:, lo:lo + cols]
        self.view.fill_(float("nan"))

    def check(self, ref, what):
        _check(self.view, ref, what)
        outside = torch.cat([self.full[:, :self.lo], self.full[:, self.lo + self.cols:]], 1)
        assert bool((outside == SENTINEL).all()), f"{what}: wrote outside its column slice"


def _ref_gemm(a, w, bias=None, rowvec=None, rows_per_batch=0, ln=None, act=0, residual=None, out_f32=False):
    acc = a.float() @ w.float().t()
    if ln is not None:
        stats, colsum = ln
        acc = acc * stats[:, 0:1] - stats[:, 1:2] * colsum
    if bias is not None:
        acc = acc + bias
    if rowvec is not None:
        acc = acc + rowvec[torch.arange(a.shape[0], device="cuda") // rows_per_batch]
    if act == 2:
        v = acc.view(acc.shape[0], -1, 2, 16)
        xv, gv = v[:, :, 0].to(BF).float(), v[:, :, 1].to(BF).float()
        acc = (xv * _gelu(gv).to(BF).float()).reshape(acc.shape[0], -1)
    elif act == 1:
        acc = F.silu(acc.to(BF).float())
    if residual is not None:
        acc = (acc if out_f32 else acc.to(BF).float()) + residual.float()
    return acc


def _with_width(lib, bn, fn):
    lib.supir_set_gemm_tile_n(bn)
    try:
        return fn()
    finally:
        lib.supir_set_gemm_tile_n(0)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("bn", [64, 128, 160, 256])
@pytest.mark.parametrize("which", ["1", "2", "sms-1", "sms+1", "2sms+1"])
def test_gemm_persistent_tile_counts(which, bn):
    """One n-tile, so the tile count is the m-tile count; the last m-tile is ragged (M not a multiple of 128)."""
    ops, lib = _ops()
    sms = _sms()
    tiles = {"1": 1, "2": 2, "sms-1": sms - 1, "sms+1": sms + 1, "2sms+1": 2 * sms + 1}[which]
    M, N, K = tiles * 128 - 37, bn, 192
    a, w = _rand((M, K), 1), _rand((N, K), 2, 1 / math.sqrt(K))
    bias, res = _randf((N,), 3, 0.2), _rand((M, N), 4)
    out = _Slice(M, N)
    _with_width(lib, bn, lambda: ops.gemm(a, w, out.view, bias=bias, residual=res))
    out.check(_ref_gemm(a, w, bias=bias, residual=res), f"gemm tiles={tiles} bn={bn}")


@pytest.mark.parametrize("bn", WIDTHS)
@pytest.mark.parametrize("N", [320, 200, 1000])
def test_gemm_ragged_n(N, bn):
    """N not a multiple of the tile width (320 at 128 or 256; 200 is not a multiple of 32, 1000 of 64)."""
    ops, lib = _ops()
    M, K = 1000, 640
    a, w = _rand((M, K), 5), _rand((N, K), 6, 1 / math.sqrt(K))
    bias, res = _randf((N,), 7, 0.2), _rand((M, N), 8)
    out = _Slice(M, N)
    _with_width(lib, bn, lambda: ops.gemm(a, w, out.view, bias=bias, residual=res))
    out.check(_ref_gemm(a, w, bias=bias, residual=res), f"gemm N={N} bn={bn}")


EPILOGUES = {
    "bias": dict(bias=True),
    "rowvec": dict(bias=True, rowvec=True),
    "ln": dict(bias=True, ln=True),
    "ln_rowvec_res": dict(bias=True, ln=True, rowvec=True, res=True),
    "silu": dict(bias=True, act=1),
    "geglu": dict(bias=True, act=2),
    "geglu_rowvec_res": dict(bias=True, rowvec=True, act=2, res=True),
    "res_slice": dict(bias=True, res=True),
    "res_odd": dict(res=True, res_odd=True),
    "f32": dict(bias=True, f32=True),
    "f32_res": dict(bias=True, res=True, f32=True),
    "out_slice": dict(bias=True, res=True, out_lo=24, out_hi=40),
    "out_slice_f32": dict(bias=True, rowvec=True, f32=True, out_lo=12, out_hi=4),
    "out_odd_ldc": dict(bias=True, res=True, out_lo=1, out_hi=2),
}


@pytest.mark.parametrize("bn", WIDTHS)
@pytest.mark.parametrize("name", list(EPILOGUES))
def test_gemm_epilogues(name, bn):
    """rows_per_batch = 300 puts image boundaries inside 128-row tiles; the residual is a column slice (ldr != n_out),
    or starts at an odd element; out_slice writes columns [lo, lo + n_out) of a wider buffer; an odd leading dimension
    makes the output rows 2-byte aligned."""
    e = EPILOGUES[name]
    ops, lib = _ops()
    M, N, K, rpb = 1100, 640, 640, 300
    act = e.get("act", 0)
    n_out = N // 2 if act == 2 else N
    a, w = _rand((M, K), 11), _rand((N, K), 12, 1 / math.sqrt(K))
    bias = _randf((N,), 13, 0.2) if e.get("bias") else None
    rowvec = _randf((M // rpb + 1, N), 14, 0.5) if e.get("rowvec") else None
    ln = None
    if e.get("ln"):
        stats = torch.stack([_randf((M,), 15).abs() + 0.5, _randf((M,), 16, 0.3)], 1).contiguous()
        ln = (stats, _randf((N,), 17, 0.5))
    res = None
    if e.get("res"):
        lo = 3 if e.get("res_odd") else 8
        res = _rand((M, n_out + 24), 18)[:, lo:lo + n_out]
    dtype = torch.float32 if e.get("f32") else BF
    out = _Slice(M, n_out, e.get("out_lo", 0), e.get("out_hi", 0), dtype)
    _with_width(lib, bn, lambda: ops.gemm(a, w, out.view, bias=bias, rowvec=rowvec, rows_per_batch=rpb if rowvec is not None else 0,
                                          residual=res, act=act, ln=ln))
    ref = _ref_gemm(a, w, bias, rowvec, rpb, ln, act, res, dtype == torch.float32)
    out.check(ref, f"gemm epilogue {name} bn={bn}")


def test_gemm_deterministic():
    ops, lib = _ops()
    M, N, K = 4000, 1280, 1280
    a, w = _rand((M, K), 21), _rand((N, K), 22, 1 / math.sqrt(K))
    bias, res = _randf((N,), 23, 0.2), _rand((M, N), 24)
    o1, o2 = torch.empty((M, N), dtype=BF, device="cuda"), torch.empty((M, N), dtype=BF, device="cuda")
    ops.gemm(a, w, o1, bias=bias, residual=res)
    ops.gemm(a, w, o2, bias=bias, residual=res)
    assert torch.equal(o1, o2)
    g1, g2 = torch.empty((M, N // 2), dtype=BF, device="cuda"), torch.empty((M, N // 2), dtype=BF, device="cuda")
    ops.gemm(a, w, g1, bias=bias, act=2)
    ops.gemm(a, w, g2, bias=bias, act=2)
    assert torch.equal(g1, g2)


# ----------------------------------------------------------------------------------------------------------------------
# convolution
# ----------------------------------------------------------------------------------------------------------------------
def _nchw(x, B, H, W):
    return x.float().view(B, H, W, -1).permute(0, 3, 1, 2)


def _nhwc(y):
    return y.permute(0, 2, 3, 1).reshape(-1, y.shape[1])


@pytest.mark.parametrize("bn", WIDTHS)
@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 13, 21, 72, 320), (3, 7, 40, 64, 200), (1, 33, 9, 128, 640)])
def test_conv3x3_ragged_rowvec_residual(B, H, W, Cin, Cout, bn):
    """H, W not multiples of the pixel patch; Cin = 72 leaves a partial 64-channel chunk; per-image vector + residual."""
    ops, lib = _ops()
    x = _rand((B * H * W, Cin), 31)
    w = _rand((Cout, Cin, 3, 3), 32, 1 / math.sqrt(9 * Cin))
    bias, rv, res = _randf((Cout,), 33, 0.2), _randf((B, Cout), 34, 0.5), _rand((B * H * W, Cout), 35)
    wp = w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous()
    out = _Slice(B * H * W, Cout)
    _with_width(lib, bn, lambda: ops.conv3x3(x, B, H, W, wp, out.view, bias=bias, rowvec=rv, residual=res))
    y = F.conv2d(_nchw(x, B, H, W), w.float(), bias, padding=1) + rv[:, :, None, None]
    out.check(_nhwc(y).to(BF).float() + res.float(), f"conv {B}x{H}x{W} {Cin}->{Cout} bn={bn}")


@pytest.mark.parametrize("bn", WIDTHS)
@pytest.mark.parametrize("pad_lo", [1, 0])
def test_conv3x3_stride2(pad_lo, bn):
    ops, lib = _ops()
    B, H, W, Cin, Cout = 2, 30, 22, 128, 320
    x = _rand((B * H * W, Cin), 41)
    w = _rand((Cout, Cin, 3, 3), 42, 1 / math.sqrt(9 * Cin))
    bias = _randf((Cout,), 43, 0.2)
    wp = w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous()
    xi = _nchw(x, B, H, W)
    y = F.conv2d(xi, w.float(), bias, stride=2, padding=1) if pad_lo else F.conv2d(F.pad(xi, (0, 1, 0, 1)), w.float(), bias, stride=2)
    out = _Slice(B * y.shape[2] * y.shape[3], Cout)
    _with_width(lib, bn, lambda: ops.conv3x3_stride2(x, B, H, W, wp, out.view, pad_lo, bias=bias))
    out.check(_nhwc(y), f"conv stride 2 pad_lo={pad_lo} bn={bn}")


@pytest.mark.parametrize("bn", WIDTHS)
def test_upsample2x_conv3x3_interleaved(bn):
    """Four sub-pixel 2x2 convolutions, each writing every second pixel of every second row of the output."""
    ops, lib = _ops()
    B, H, W, Cin, Cout = 2, 11, 17, 128, 320
    x = _rand((B * H * W, Cin), 51)
    w = _rand((Cout, Cin, 3, 3), 52, 1 / math.sqrt(9 * Cin))
    bias = _randf((Cout,), 53, 0.2)
    wfold = ops.fold_upsample_weights(w)
    out = _Slice(B * 4 * H * W, Cout)
    _with_width(lib, bn, lambda: ops.upsample2x_conv3x3(x, B, H, W, wfold, out.view, bias=bias))
    y = F.conv2d(F.interpolate(_nchw(x, B, H, W), scale_factor=2, mode="nearest"), w.float(), bias, padding=1)
    out.check(_nhwc(y), f"upsample2x conv bn={bn}")
