"""GPU tests of the GEMM / implicit-GEMM convolution kernel's staged epilogue (results written to shared memory and stored,
with the residual loaded, by TMA) against its direct epilogue (global stores from the accumulator fragment).

A launch takes the staged epilogue when its 16-bit output and residual have 16-byte aligned base pointers and row strides.
Each case runs the same operands twice: once into an aligned column slice (staged) and once into a slice at column offset 1
of a buffer with an odd leading dimension (direct). The epilogue arithmetic and its rounding points are shared, so the two
outputs must be bit-identical. Both are written into NaN-filled views of buffers whose other columns hold a sentinel, so a
missed or stray TMA store fails. The GEMM cases have at least 2 SMs + 1 tiles, so every staging buffer is reused and the
ping-pong consumers get unequal tile counts."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
SENTINEL = 7.0
WIDTHS = (64, 128, 160, 256)
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


def _staged_vs_direct(lib, bn, rows, cols, dtype, run, what):
    """run(out_view) launches into `out_view`; staged: aligned slice (ldc = cols + 16), direct: odd offset and ldc."""
    staged, direct = _Slice(rows, cols, 8, 8, dtype), _Slice(rows, cols, 1, 2, dtype)
    lib.supir_set_gemm_tile_n(bn)
    try:
        run(staged.view)
        run(direct.view)
    finally:
        lib.supir_set_gemm_tile_n(0)
    torch.cuda.synchronize()
    assert not bool(torch.isnan(direct.view.float()).any()), f"{what}: direct path left elements unwritten"
    assert not bool(torch.isnan(staged.view.float()).any()), f"{what}: staged path left elements unwritten"
    assert staged.outside_ok() and direct.outside_ok(), f"{what}: wrote outside the output slice"
    ndiff = int((staged.view != direct.view).sum())
    assert ndiff == 0, f"{what}: {ndiff} elements differ between the staged and the direct epilogue"


EPILOGUES = {
    "plain": dict(),
    "bias": dict(bias=True),
    "rowvec": dict(bias=True, rowvec=True),
    "ln": dict(bias=True, ln=True),
    "ln_rowvec_res": dict(bias=True, ln=True, rowvec=True, res=True),
    "silu": dict(bias=True, act=1),
    "silu_res": dict(bias=True, act=1, res=True),
    "geglu": dict(bias=True, act=2),
    "geglu_rowvec_res": dict(bias=True, rowvec=True, act=2, res=True),
    "res": dict(bias=True, res=True),
}


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("bn", WIDTHS)
@pytest.mark.parametrize("name", list(EPILOGUES))
def test_gemm_staged_equals_direct(name, bn, dt):
    """N = 608 leaves a ragged last n-tile at every width (and a partial 32-column slab at 64 / 128 / 256); M is ragged;
    rows_per_batch = 300 puts image boundaries inside tiles; the residual is a column slice of a wider tensor."""
    e = EPILOGUES[name]
    ops, lib = _ops()
    dtype = DTYPES[dt]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    act = e.get("act", 0)
    N, K, rpb = (640 if act == 2 else 608), 192, 300
    n_out = N // 2 if act == 2 else N
    m_tiles = -(-(2 * sms + 1) // -(-N // bn))
    M = m_tiles * 128 - 37
    a, w = _randf((M, K), 11).to(dtype), _randf((N, K), 12, 1 / math.sqrt(K)).to(dtype)
    bias = _randf((N,), 13, 0.2) if e.get("bias") else None
    rowvec = _randf((M // rpb + 1, N), 14, 0.5) if e.get("rowvec") else None
    ln = None
    if e.get("ln"):
        stats = torch.stack([_randf((M,), 15).abs() + 0.5, _randf((M,), 16, 0.3)], 1).contiguous()
        ln = (stats, _randf((N,), 17, 0.5))
    res = _randf((M, n_out + 24), 18).to(dtype)[:, 8:8 + n_out] if e.get("res") else None
    _staged_vs_direct(lib, bn, M, n_out, dtype,
                      lambda out: ops.gemm(a, w, out, bias=bias, rowvec=rowvec, rows_per_batch=rpb if rowvec is not None else 0,
                                           residual=res, act=act, ln=ln),
                      f"gemm {name} bn={bn} {dt}")


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("bn", WIDTHS)
def test_gemm_staged_misaligned_residual(bn, dt):
    """A residual at an odd element address takes the direct path; the same values from an aligned copy take the staged one."""
    ops, lib = _ops()
    dtype = DTYPES[dt]
    M, N, K = 3000, 640, 256
    a, w = _randf((M, K), 21).to(dtype), _randf((N, K), 22, 1 / math.sqrt(K)).to(dtype)
    bias = _randf((N,), 23, 0.2)
    res_odd = _randf((M, N + 8), 24).to(dtype)[:, 3:3 + N]
    res_al = res_odd.contiguous()
    outs = []
    lib.supir_set_gemm_tile_n(bn)
    try:
        for r in (res_al, res_odd):
            o = torch.full((M, N), float("nan"), dtype=dtype, device="cuda")
            ops.gemm(a, w, o, bias=bias, residual=r)
            outs.append(o)
    finally:
        lib.supir_set_gemm_tile_n(0)
    assert not bool(torch.isnan(outs[0].float()).any())
    assert torch.equal(outs[0], outs[1]), f"bn={bn} {dt}: staged and direct residual epilogues differ"


def _packed(w):
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1).contiguous()


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("bn", WIDTHS)
@pytest.mark.parametrize("B,H,W,Cin,Cout", [(3, 70, 45, 64, 320), (2, 13, 21, 72, 200), (1, 5, 150, 64, 96), (2, 33, 9, 128, 640)])
def test_conv3x3_staged_equals_direct(B, H, W, Cin, Cout, bn, dt):
    """Ragged patches (H, W not multiples of TH, TW; W = 150 takes the 128 x 1 patch), per-image vector + residual."""
    ops, lib = _ops()
    dtype = DTYPES[dt]
    x = _randf((B * H * W, Cin), 31).to(dtype)
    wp = _packed(_randf((Cout, Cin, 3, 3), 32, 1 / math.sqrt(9 * Cin)).to(dtype))
    bias, rv, res = _randf((Cout,), 33, 0.2), _randf((B, Cout), 34, 0.5), _randf((B * H * W, Cout), 35).to(dtype)
    _staged_vs_direct(lib, bn, B * H * W, Cout, dtype,
                      lambda out: ops.conv3x3(x, B, H, W, wp, out, bias=bias, rowvec=rv, residual=res),
                      f"conv {B}x{H}x{W} {Cin}->{Cout} bn={bn} {dt}")


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("bn", WIDTHS)
@pytest.mark.parametrize("pad_lo", [1, 0])
def test_conv3x3_stride2_staged_equals_direct(pad_lo, bn, dt):
    ops, lib = _ops()
    dtype = DTYPES[dt]
    B, H, W, Cin, Cout = 2, 30, 22, 128, 320
    x = _randf((B * H * W, Cin), 41).to(dtype)
    wp = _packed(_randf((Cout, Cin, 3, 3), 42, 1 / math.sqrt(9 * Cin)).to(dtype))
    bias = _randf((Cout,), 43, 0.2)
    Ho = (H + 2 * pad_lo - 3) // 2 + 1 if pad_lo else (H - 2) // 2 + 1
    Wo = (W + 2 * pad_lo - 3) // 2 + 1 if pad_lo else (W - 2) // 2 + 1
    _staged_vs_direct(lib, bn, B * Ho * Wo, Cout, dtype,
                      lambda out: ops.conv3x3_stride2(x, B, H, W, wp, out, pad_lo, bias=bias),
                      f"conv stride 2 pad_lo={pad_lo} bn={bn} {dt}")


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("bn", WIDTHS)
def test_upsample2x_conv3x3_staged_equals_direct(bn, dt):
    """Four sub-pixel convolutions, each storing every second pixel of every second output row."""
    ops, lib = _ops()
    dtype = DTYPES[dt]
    B, H, W, Cin, Cout = 2, 11, 17, 128, 320
    x = _randf((B * H * W, Cin), 51).to(dtype)
    wfold = ops.fold_upsample_weights(_randf((Cout, Cin, 3, 3), 52, 1 / math.sqrt(9 * Cin)), dtype)
    bias = _randf((Cout,), 53, 0.2)
    _staged_vs_direct(lib, bn, B * 4 * H * W, Cout, dtype,
                      lambda out: ops.upsample2x_conv3x3(x, B, H, W, wfold, out, bias=bias),
                      f"upsample2x conv bn={bn} {dt}")
