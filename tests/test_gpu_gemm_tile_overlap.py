"""GPU tests of the 160-wide GEMM / implicit-GEMM convolution tile (the width the step's short-k-loop shapes take) and its
epilogue, which applies each column operand (folded LayerNorm column sums, bias, per-image vector) in a pass of its own.

Every case runs the same operands through the staged epilogue (aligned output slice: TMA stores, TMA-loaded residual) and
the direct one (output at column offset 1 of a buffer with an odd leading dimension), both into NaN-filled views whose
surrounding columns hold a sentinel. The two must be bit-identical (shared arithmetic and rounding points), and the staged
output must match plain PyTorch fp32 maths on the same 16-bit operands (tolerance 2e-2 + 2e-2 |ref|), so a dropped tile
(NaN left), a stray store (sentinel overwritten) or a tile written to another tile's place (values off by O(1)) fails.
The tile counts cover an odd number of tiles per persistent CTA, unequal counts across CTAs, a launch of one tile, and
ragged last m- and n-tiles."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
BN = 160
SENTINEL = 7.0
DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}


def _ops():
    from supir_b200 import _native, ops
    return ops, _native.load()


def _randf(shape, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(shape, generator=g, device="cuda") * scale


class _Slice:
    def __init__(self, rows, cols, lo, hi, dtype):
        self.full = torch.full((rows, lo + cols + hi), SENTINEL, dtype=dtype, device="cuda")
        self.lo, self.cols = lo, cols
        self.view = self.full[:, lo:lo + cols]
        self.view.fill_(float("nan"))

    def outside_ok(self):
        outside = torch.cat([self.full[:, :self.lo], self.full[:, self.lo + self.cols:]], 1)
        return bool((outside == SENTINEL).all())


def _run_both(lib, rows, cols, dtype, run, ref, what):
    """run(out_view) launches at width 160 into `out_view`: staged (aligned slice whose row stride is a multiple of 8
    elements, so TMA can address it) and direct (odd offset and ldc)."""
    staged, direct = _Slice(rows, cols, 8, 8 + (-cols) % 8, dtype), _Slice(rows, cols, 1, 2, dtype)   # staged: ldc % 8 == 0
    lib.supir_set_gemm_tile_n(BN)
    try:
        run(staged.view)
        run(direct.view)
    finally:
        lib.supir_set_gemm_tile_n(0)
    torch.cuda.synchronize()
    for name, s in (("staged", staged), ("direct", direct)):
        assert not bool(torch.isnan(s.view.float()).any()), f"{what}: {name} path left elements unwritten"
        assert s.outside_ok(), f"{what}: {name} path wrote outside the output slice"
    ndiff = int((staged.view != direct.view).sum())
    assert ndiff == 0, f"{what}: {ndiff} elements differ between the staged and the direct epilogue"
    err = (staged.view.float() - ref).abs()
    nbad = int((err > 2e-2 + 2e-2 * ref.abs()).sum())
    assert nbad == 0, f"{what}: {nbad} elements out of tolerance against fp32 maths, max err {float(err.max()):.4g}"


def _ref_gemm(a, w, dtype, bias=None, rowvec=None, rows_per_batch=0, ln=None, act=0, residual=None):
    acc = a.float() @ w.float().t()
    if ln is not None:
        acc = acc * ln[0][:, 0:1] - ln[0][:, 1:2] * ln[1]
    if bias is not None:
        acc = acc + bias
    if rowvec is not None:
        acc = acc + rowvec[torch.arange(a.shape[0], device="cuda") // rows_per_batch]
    if act == 1:
        acc = F.silu(acc.to(dtype).float())
    if residual is not None:
        acc = acc.to(dtype).float() + residual.float()
    return acc


EPILOGUES = {
    "bias": dict(bias=True),
    "rowvec": dict(rowvec=True),
    "bias_rowvec": dict(bias=True, rowvec=True),
    "ln": dict(bias=True, ln=True),
    "ln_rowvec_res": dict(bias=True, ln=True, rowvec=True, res=True),
    "silu": dict(bias=True, act=1),
    "silu_rowvec_res": dict(bias=True, rowvec=True, act=1, res=True),
    "res": dict(res=True),
    "bias_res": dict(bias=True, res=True),
}


def _tiles(which, n_tiles):
    """m-tile count for a launch of `n_tiles` n-tiles: every CTA 3 tiles (odd), 2 or 3 tiles per CTA, or one tile."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return {"odd": -(-3 * sms // n_tiles), "mixed": -(-(2 * sms + 1) // n_tiles), "single": 1}[which]


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("which", ["odd", "mixed", "single"])
@pytest.mark.parametrize("name", list(EPILOGUES))
def test_gemm_width160(name, which, dt):
    """N = 608 = 3 x 160 + 128 leaves a ragged last n-tile (152 for one tile: its last 32-column slab is clipped); M ends 37
    rows into its last m-tile; the per-image vector's images change inside m-tiles (rows_per_batch 300, or 37 for one
    tile)."""
    e = EPILOGUES[name]
    ops, lib = _ops()
    dtype = DTYPES[dt]
    N = 152 if which == "single" else 608
    M = _tiles(which, -(-N // BN)) * 128 - 37
    K, rpb = 192, (37 if which == "single" else 300)
    a, w = _randf((M, K), 11).to(dtype), _randf((N, K), 12, 1 / math.sqrt(K)).to(dtype)
    bias = _randf((N,), 13, 0.2) if e.get("bias") else None
    rowvec = _randf((M // rpb + 1, N), 14, 0.5) if e.get("rowvec") else None
    ln = None
    if e.get("ln"):
        ln = (torch.stack([_randf((M,), 15).abs() + 0.5, _randf((M,), 16, 0.3)], 1).contiguous(), _randf((N,), 17, 0.5))
    res = _randf((M, N + 24 + (-N) % 8), 18).to(dtype)[:, 8:8 + N] if e.get("res") else None   # row stride % 8 == 0
    act = e.get("act", 0)
    ref = _ref_gemm(a, w, dtype, bias, rowvec, rpb, ln, act, res)
    _run_both(lib, M, N, dtype,
              lambda out: ops.gemm(a, w, out, bias=bias, rowvec=rowvec, rows_per_batch=rpb if rowvec is not None else 0,
                                   residual=res, act=act, ln=ln),
              ref, f"gemm {name} {which} {dt}")


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("bn", [0, 64, 128, 160, 256])
def test_gemm_output_edge_inside_16_bytes(bn, dt):
    """150 output columns end inside a 16-byte chunk, so the launch takes the direct epilogue even into an aligned slice:
    nothing may land in the slice's right-hand neighbours."""
    ops, lib = _ops()
    dtype = DTYPES[dt]
    M, N, K = 1000, 150, 192
    a, w = _randf((M, K), 61).to(dtype), _randf((N, K), 62, 1 / math.sqrt(K)).to(dtype)
    bias, res = _randf((N,), 63, 0.2), _randf((M, N + 26), 64).to(dtype)[:, 8:8 + N]
    out = _Slice(M, N, 8, 10, dtype)
    lib.supir_set_gemm_tile_n(bn)
    try:
        ops.gemm(a, w, out.view, bias=bias, residual=res)
    finally:
        lib.supir_set_gemm_tile_n(0)
    torch.cuda.synchronize()
    assert out.outside_ok(), f"bn={bn} {dt}: wrote past the output's last column"
    ref = _ref_gemm(a, w, dtype, bias=bias, residual=res)
    err = (out.view.float() - ref).abs()
    assert int((err > 2e-2 + 2e-2 * ref.abs()).sum()) == 0, f"bn={bn} {dt}: max err {float(err.max()):.4g}"


def _nchw(x, B, H, W):
    return x.float().view(B, H, W, -1).permute(0, 3, 1, 2)


def _nhwc(y):
    return y.permute(0, 2, 3, 1).reshape(-1, y.shape[1])


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("B,H,W,Cin,Cout", [(3, 70, 45, 64, 320), (2, 13, 21, 72, 200), (1, 8, 16, 64, 96)])
def test_conv3x3_width160(B, H, W, Cin, Cout, dt):
    """Ragged pixel patches, a ragged last n-tile, per-image vector and residual; 1 x 8 x 16 is a single tile."""
    ops, lib = _ops()
    dtype = DTYPES[dt]
    x = _randf((B * H * W, Cin), 31).to(dtype)
    w = _randf((Cout, Cin, 3, 3), 32, 1 / math.sqrt(9 * Cin)).to(dtype)
    bias, rv, res = _randf((Cout,), 33, 0.2), _randf((B, Cout), 34, 0.5), _randf((B * H * W, Cout), 35).to(dtype)
    wp = w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous()
    y = F.conv2d(_nchw(x, B, H, W), w.float(), bias, padding=1) + rv[:, :, None, None]
    ref = _nhwc(y).to(dtype).float() + res.float()
    _run_both(lib, B * H * W, Cout, dtype, lambda out: ops.conv3x3(x, B, H, W, wp, out, bias=bias, rowvec=rv, residual=res),
              ref, f"conv {B}x{H}x{W} {Cin}->{Cout} {dt}")


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("pad_lo", [1, 0])
def test_conv3x3_stride2_width160(pad_lo, dt):
    ops, lib = _ops()
    dtype = DTYPES[dt]
    B, H, W, Cin, Cout = 2, 30, 22, 128, 320
    x = _randf((B * H * W, Cin), 41).to(dtype)
    w = _randf((Cout, Cin, 3, 3), 42, 1 / math.sqrt(9 * Cin)).to(dtype)
    bias = _randf((Cout,), 43, 0.2)
    wp = w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous()
    xi = _nchw(x, B, H, W)
    y = F.conv2d(xi, w.float(), bias, stride=2, padding=1) if pad_lo else F.conv2d(F.pad(xi, (0, 1, 0, 1)), w.float(), bias, stride=2)
    _run_both(lib, B * y.shape[2] * y.shape[3], Cout, dtype, lambda out: ops.conv3x3_stride2(x, B, H, W, wp, out, pad_lo, bias=bias),
              _nhwc(y), f"conv stride 2 pad_lo={pad_lo} {dt}")


@pytest.mark.parametrize("dt", list(DTYPES))
def test_upsample2x_conv3x3_width160(dt):
    """Four sub-pixel convolutions, each storing every second pixel of every second output row."""
    ops, lib = _ops()
    dtype = DTYPES[dt]
    B, H, W, Cin, Cout = 2, 11, 17, 128, 320
    x = _randf((B * H * W, Cin), 51).to(dtype)
    w = _randf((Cout, Cin, 3, 3), 52, 1 / math.sqrt(9 * Cin))
    bias = _randf((Cout,), 53, 0.2)
    wfold = ops.fold_upsample_weights(w, dtype)
    y = F.conv2d(F.interpolate(_nchw(x, B, H, W), scale_factor=2, mode="nearest"), w.to(dtype).float(), bias, padding=1)
    _run_both(lib, B * 4 * H * W, Cout, dtype, lambda out: ops.upsample2x_conv3x3(x, B, H, W, wfold, out, bias=bias),
              _nhwc(y), f"upsample2x conv {dt}")
