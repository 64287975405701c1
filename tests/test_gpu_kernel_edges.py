"""The non-GEMM kernels against fp64 at their launch-path edges, and the bit-invariance that sharding relies on.

Method. Inputs are fp32 values that are exact in the storage type E (bf16 or fp16). The reference is computed in fp64 on the
device, with the kernel's documented rounding points to E applied explicitly. Each element must satisfy

    |got - ref| <= n * ulp_E(ref) + c * 2^-24 * mag

where n counts the rounding points that can flip, and `mag` is the fp64 sum of the magnitudes the kernel combined in fp32 (the
standard gamma_n * sum|terms| bound), so results near zero are not held to a relative bound fp32 cannot meet. On top of that,
the fraction of elements that differ from the correctly rounded reference must stay small: that is what catches a systematic
1e-4-relative error that no per-element bound sees. Outputs go into NaN-filled views of wider buffers whose 16-byte borders
hold a sentinel, so a missed or stray store fails, and operands use leading dimensions larger than their width.

The CPU stand-ins of tests/cpu_ops.py, which the CPU drop-in tests run instead of the kernels, are held to the same bounds on
the same inputs (the tensor-core GEMM to the GEMM-class tolerance).

The last part checks that results do not depend on the GEMM tile width or on which other batch rows share the launch:
DESIGN.md section 5 promises that a sharded run is bit-identical to the single-GPU run."""
import math

import pytest
import torch
import torch.nn.functional as F

import cpu_ops

SENTINEL = 7.0
U = 2.0 ** -24                                   # fp32 unit roundoff
DT = {"bf16": torch.bfloat16, "fp16": torch.float16}
# Bounds on the fraction of outputs that differ from the correctly rounded fp64 value. Set from H100 runs (largest measured
# over each test's cases, in brackets) with margin; fp16 has 3 more mantissa bits, so the same fp32 error flips more roundings.
FRAC = {  # kernel: (bf16, fp16)
    "groupnorm": (5e-3, 2e-2),        # measured (2.1e-3, 9.0e-3): small groups, where the statistics' fp32 error shows
    "layernorm": (1e-3, 4e-3),        # (4.6e-5, 7.8e-4)
    "small_cin": (2e-3, 1e-2),        # (8.8e-5, 3.7e-3)
    "small_cin_res": (2e-3, 2e-3),    # (9.0e-5, 2.7e-4)
    "small_cout": (3e-3, 1e-2),       # (7.1e-4, 2.8e-3)
    "conv1x1": (2e-3, None),          # (5.7e-4, -)
    "softmax": (1e-3, None),          # (1.0e-4, -)
    "linear_small_m": (2e-3, 1.5e-2), # (4.7e-4, 7.0e-3): five rounding points in a chain, so an early flip carries through
    "attention_small": (2e-3, None),  # (2.7e-4, -)
}
_FMT = {torch.bfloat16: (8, -126), torch.float16: (11, -14), torch.float32: (24, -126)}   # (precision bits, min exponent)


# ------------------------------------------------------------------------------------------------------------------
# helpers (the ulp helper has a CPU test)
# ------------------------------------------------------------------------------------------------------------------
def ulp(ref, dtype):
    """Spacing of `dtype` at |ref| (elementwise, fp64): 2^(e - p + 1) for |ref| in [2^e, 2^(e+1)), and the subnormal
    spacing 2^(emin - p + 1) below the normal range (zero included)."""
    p, emin = _FMT[dtype]
    a = ref.double().abs()
    _, e = torch.frexp(a)                         # a = m * 2^e, m in [0.5, 1); frexp(0) gives e = 0
    e = torch.where(a == 0, float(emin), torch.clamp(e.double() - 1, min=emin))
    return torch.exp2(e - (p - 1))


def check(got, ref, dtype, n=1.0, err=None, frac=None, mask=None, what=""):
    """Per-element bound n * ulp_dtype(ref) + err (err: fp64 tensor of the fp32 arithmetic's error bound, or None), and the
    fraction of elements (under `mask`) that differ from ref rounded to dtype at most `frac`. Returns that fraction."""
    g, r = got.double(), ref.double()
    tol = n * ulp(r, dtype)
    if err is not None:
        tol = tol + err
    bad = ~((g - r).abs() <= tol)                 # NaN in got fails
    nbad = int(bad.sum())
    if nbad:
        i = int(bad.flatten().nonzero()[0])
        raise AssertionError(f"{what}: {nbad} of {g.numel()} elements out of bound; first at {i}: got {g.flatten()[i].item()!r} "
                             f"ref {r.flatten()[i].item()!r} tol {tol.flatten()[i].item():.3g}")
    ne = got.to(dtype) != ref.to(dtype)
    if mask is not None:
        ne = ne[mask.expand_as(ne)]
    f = float(ne.double().mean()) if ne.numel() else 0.0
    print(f"{what}: {f:.2e} of the elements differ from the correctly rounded fp64 value")
    if frac is not None:
        assert f <= frac, f"{what}: {f:.3e} of the elements differ from the correctly rounded fp64 value (bound {frac:.1e})"
    return f


def test_ulp_helper_on_hand_picked_values():
    """No GPU: neighbours in bf16 / fp16 differ by exactly one ulp, zeros and subnormals get the subnormal spacing."""
    bf, hf = torch.bfloat16, torch.float16
    for dt in (bf, hf):
        p, emin = _FMT[dt]
        for v in (1.0, 1.5, -3.0, 0.1, 1000.0, 2.0 ** emin, 2.0 ** (emin - 3), 0.0):
            x = torch.tensor([v], dtype=dt)
            nxt = (x.view(torch.int16) + (1 if v >= 0 else -1)).view(dt)      # the next value away from zero, by bit pattern
            assert float(ulp(x.double(), dt)) == abs(float(nxt.double() - x.double())), (dt, v)
    assert float(ulp(torch.tensor([1.0]), bf)) == 2.0 ** -7
    assert float(ulp(torch.tensor([1.0 - 2 ** -9]), bf)) == 2.0 ** -8     # just below a power of two: the finer spacing
    assert float(ulp(torch.tensor([65504.0]), hf)) == 32.0
    assert float(ulp(torch.tensor([0.0]), hf)) == 2.0 ** -24              # fp16 subnormal spacing
    assert float(ulp(torch.tensor([3e-8]), hf)) == 2.0 ** -24
    assert float(ulp(torch.tensor([0.0]), bf)) == 2.0 ** -133
    assert float(ulp(torch.tensor([-2.0 ** -130]), bf)) == 2.0 ** -133
    # check(): exactly one ulp passes at n = 1, two do not; NaN fails
    r = torch.tensor([1.0, 2.0, -0.5], dtype=torch.float64)
    check(r + torch.tensor([2 ** -7, 0, 0]), r, bf, frac=1.0)
    with pytest.raises(AssertionError):
        check(r + torch.tensor([2 ** -6, 0, 0]), r, bf)
    with pytest.raises(AssertionError):
        check(torch.tensor([math.nan, 2.0, -0.5]), r, bf)


def _cpu(*ts):
    """CPU copies of the operands, for the stand-ins of tests/cpu_ops.py."""
    return [t.cpu() if isinstance(t, torch.Tensor) else t for t in ts]


def _ops():
    from supir_b200 import _native, ops
    return ops, _native.load()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _randn(shape, seed, scale=1.0, dtype=None):
    t = torch.randn(shape, generator=_gen(seed), device="cuda") * scale
    return t if dtype is None else t.to(dtype)


def _strided(t, extra=8):
    """The same values as a column slice of a wider buffer (leading dimension > width)."""
    buf = torch.full((t.shape[0], t.shape[1] + extra), SENTINEL, dtype=t.dtype, device=t.device)
    buf[:, :t.shape[1]] = t
    return buf[:, :t.shape[1]]


class _Out:
    """NaN-filled [rows, cols] view of a buffer with SENTINEL columns on both sides: `lo` elements on the left (16 bytes by
    default, so vector stores stay aligned) and at least 16 bytes on the right, the row stride rounded to 16 bytes."""

    def __init__(self, rows, cols, dtype, lo=None):
        es = torch.empty((), dtype=dtype).element_size()
        v = 16 // es
        lo = v if lo is None else lo
        ld = lo + (cols + v - 1) // v * v + v
        self.full = torch.full((rows, ld), SENTINEL, dtype=dtype, device="cuda")
        self.lo, self.cols = lo, cols
        self.view = self.full[:, lo:lo + cols]
        self.view.fill_(float("nan"))

    def done(self, what):
        torch.cuda.synchronize()
        assert not bool(torch.isnan(self.view.float()).any()), f"{what}: elements left unwritten"
        out = torch.cat([self.full[:, :self.lo], self.full[:, self.lo + self.cols:]], 1)
        assert bool((out == SENTINEL).all()), f"{what}: wrote outside the output view"
        return self.view


class _Flat:
    """A contiguous NaN-filled tensor of `shape` inside a flat buffer with 16 bytes of SENTINEL on each side."""

    def __init__(self, shape, dtype):
        v = 16 // torch.empty((), dtype=dtype).element_size()
        n = math.prod(shape)
        self.full = torch.full((n + 2 * v,), SENTINEL, dtype=dtype, device="cuda")
        self.v, self.n = v, n
        self.view = self.full[v:v + n].view(shape)
        self.view.fill_(float("nan"))

    def done(self, what):
        torch.cuda.synchronize()
        assert not bool(torch.isnan(self.view.float()).any()), f"{what}: elements left unwritten"
        assert self.borders_ok(), f"{what}: wrote outside the output"
        return self.view

    def borders_ok(self):
        return bool((self.full[:self.v] == SENTINEL).all()) and bool((self.full[self.v + self.n:] == SENTINEL).all())


class _Canvas:
    """fp32 NCHW window [B, C, h, w] at offset (oy, ox) of a larger SENTINEL canvas, NaN-filled (strides ob != C*h*w)."""

    def __init__(self, B, C, h, w, oy=3, ox=5, ey=4, ex=6):
        self.full = torch.full((B, C, h + oy + ey, w + ox + ex), SENTINEL, device="cuda")
        self.sl = (slice(None), slice(None), slice(oy, oy + h), slice(ox, ox + w))
        self.view = self.full[self.sl]
        self.view.fill_(float("nan"))

    def done(self, what):
        torch.cuda.synchronize()
        assert not bool(torch.isnan(self.view).any()), f"{what}: elements left unwritten"
        m = torch.ones_like(self.full, dtype=torch.bool)
        m[self.sl] = False
        assert bool((self.full[m] == SENTINEL).all()), f"{what}: wrote outside the crop window"
        return self.view


def _silu64(x):
    return x / (1 + torch.exp(-x))


# ------------------------------------------------------------------------------------------------------------------
# GroupNorm statistics / apply, tiled-VAE merge, ZeroSFT
# ------------------------------------------------------------------------------------------------------------------
def _gn_stats_shape(HW, C):
    """(pixel lanes kp, pixels per block, blocks per image) of supir_groupnorm_stats (gn_launch_shape in norm.cu)."""
    cv = C // 8
    kp = max(1, 512 // cv)
    ppb = max(kp * 16, 64)
    cap = (HW + 591) // 592
    if ppb < cap:
        ppb = (cap + kp - 1) // kp * kp
    return kp, ppb, -(-HW // ppb)


def _gn_input(B, HW, C, dtype, seed):
    """Per-group means / scales: mostly N(0.5, 2); group 3 has variance ~1e-4 (eps 1e-5 vs 1e-6 matters there); group 5 has
    |mean| / std = 30 (cancellation in E[x^2] - mean^2)."""
    cpg = C // 32
    mean = torch.full((C,), 0.5, device="cuda")
    std = torch.full((C,), 2.0, device="cuda")
    std[3 * cpg:4 * cpg] = 0.01
    mean[5 * cpg:6 * cpg], std[5 * cpg:6 * cpg] = -30.0, 1.0
    x = (_randn((B * HW, C), seed) * std + mean).to(dtype)
    return _strided(x, 8)


def _gn_reference(x, B, HW, C, sums_err_c):
    """fp64 per-(image, group) mean / biased variance, and bounds on the fp32 partial sums' error: the mean's error and the
    relative error of the variance (both from sums_err_c * 2^-24 * sum|terms|)."""
    xd = x.double().view(B, HW, 32, C // 32)
    cnt = HW * (C // 32)
    s, q, a = xd.sum((1, 3)), (xd * xd).sum((1, 3)), xd.abs().sum((1, 3))
    m = s / cnt
    v = (q / cnt - m * m).clamp(min=0)
    dm = sums_err_c * U * a / cnt
    dv = sums_err_c * U * (q / cnt + 2 * m.abs() * a / cnt)
    return s, q, a, m, v, dm, dv


def _gn_expected(x, B, HW, C, m, v, dm, dv, gamma, beta, eps, silu):
    """fp64 GroupNorm (+SiLU) and its error bound: fp32 scale / shift arithmetic (c * 2^-24 * mag) plus the statistics' error."""
    xd = x.double().view(B, HW, 32, C // 32)
    g, b = gamma.double().view(32, -1), beta.double().view(32, -1)
    rstd = 1.0 / torch.sqrt(v + eps)
    z = (xd - m[:, None, :, None]) * rstd[:, None, :, None] * g + b
    mag = (xd.abs() + m.abs()[:, None, :, None]) * rstd[:, None, :, None] * g.abs() + b.abs()
    k = (dv / (2 * (v + eps)))[:, None, :, None]
    err = 16 * U * mag + g.abs() * rstd[:, None, :, None] * ((xd - m[:, None, :, None]).abs() * k + dm[:, None, :, None])
    if silu:
        z, err = _silu64(z), 1.1 * err + 8 * U * z.abs()
    return z.reshape(B * HW, C), err.reshape(B * HW, C)


# HW large enough for the 592-block cap and more blocks than the final reduction has lanes: C = 128 at 310 k px, C = 512 at
# 80 k px (the VAE's tile sizes); C / 32 not a multiple of 8 (96, 320, 960, 2560) puts groups inside a channel vector
GN_CASES = [(96, 700, 1e-6, True), (128, 310_000, 1e-6, True), (320, 3000, 1e-5, True), (512, 80_000, 1e-6, False),
            (960, 130, 1e-5, False), (1920, 64, 1e-5, True), (2560, 40, 1e-5, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("dt", list(DT))
@pytest.mark.parametrize("C,HW,eps,silu", GN_CASES)
def test_groupnorm_stats_and_apply_vs_fp64(C, HW, eps, silu, dt):
    ops, _ = _ops()
    dtype, B = DT[dt], 2
    kp, ppb, nblk = _gn_stats_shape(HW, C)
    if HW > 592 * max(kp * 16, 64):
        assert nblk > 16, "the case must reach the final reduction's second lane step"
    x = _gn_input(B, HW, C, dtype, 100 + C)
    gamma, beta = _randn((C,), 2) * 0.3 + 1, _randn((C,), 3) * 0.3
    sums = torch.full((ops.groupnorm_ws_size(B, HW, C),), math.nan, dtype=torch.float64, device="cuda")
    ops.groupnorm_stats(x, B, HW, sums)
    c_sum = ppb // kp + kp + 4                     # fp32 adds per thread (pixel chunk) + across the kp pixel lanes
    s, q, a, m, v, dm, dv = _gn_reference(x, B, HW, C, c_sum)
    got = sums[:B * 64].view(B, 32, 2)
    xd2 = (x.double() ** 2).view(B, HW, 32, -1).sum((1, 3))
    assert bool(((got[..., 0] - s).abs() <= c_sum * U * a).all()), f"GN sums C={C} HW={HW}"
    assert bool(((got[..., 1] - q).abs() <= c_sum * U * xd2).all()), f"GN sums of squares C={C} HW={HW}"
    out = _Out(B * HW, C, dtype)
    ops.groupnorm_apply(x, B, HW, out.view, gamma, beta, eps, silu, sums=sums)
    y = out.done(f"GN apply C={C}")
    ref, err = _gn_expected(x, B, HW, C, m, v, dm, dv, gamma, beta, eps, silu)
    plain = torch.ones(C, dtype=torch.bool, device="cuda")
    plain[5 * (C // 32):6 * (C // 32)] = False     # the offset group's statistics error moves whole groups of roundings
    check(y, ref, dtype, 1, err, frac=FRAC["groupnorm"][dtype == torch.float16], mask=plain[None], what=f"GN apply C={C} HW={HW} {dt}")
    xc, gc, bc = _cpu(x, gamma, beta)
    ws = cpu_ops.groupnorm_stats(xc, B, HW, torch.zeros(cpu_ops.groupnorm_ws_size(B, HW, C), dtype=torch.float64))
    assert bool(((ws[:B * 64].view(B, 32, 2)[..., 0].cuda() - s).abs() <= c_sum * U * a).all()), "stand-in GN sums"
    ys = cpu_ops.groupnorm_apply(xc, B, HW, torch.empty(B * HW, C, dtype=dtype), gc, bc, eps, silu, sums=ws)
    check(ys.cuda(), ref, dtype, 1, err, frac=FRAC["groupnorm"][dtype == torch.float16], mask=plain[None], what=f"stand-in GN apply C={C} {dt}")


@pytest.mark.gpu
@pytest.mark.parametrize("dt", list(DT))
@pytest.mark.parametrize("C", [96, 320, 512])
def test_groupnorm_merge_tiles_and_explicit_statistics(C, dt):
    """Tiled VAE: per-tile (mean, var) merged with unequal pixel weights (tilevae's weighted mean of means and of vars), then
    GroupNorm from the explicit mean / var. The apply is checked against fp64 from the fp32 statistics it was given."""
    ops, _ = _ops()
    dtype, B, HW = DT[dt], 2, 4000
    x = _gn_input(B, HW, C, dtype, 7 + C)
    xd = x.double().view(B, HW, 32, C // 32)
    bounds = [0, 700, 2900, HW]
    tm = torch.stack([xd[:, p0:p1].mean((1, 3)) for p0, p1 in zip(bounds, bounds[1:])]).float().reshape(3, -1)
    tv = torch.stack([xd[:, p0:p1].var((1, 3), unbiased=False) for p0, p1 in zip(bounds, bounds[1:])]).float().reshape(3, -1)
    n = torch.tensor([p1 - p0 for p0, p1 in zip(bounds, bounds[1:])], dtype=torch.float64)
    w = (n / n.max() / (n / n.max()).sum()).float().cuda()
    mean, var = torch.full((B * 32,), math.nan, device="cuda"), torch.full((B * 32,), math.nan, device="cuda")
    ops.groupnorm_merge_tiles(tm.contiguous(), tv.contiguous(), w, mean, var)
    for got, t in ((mean, tm), (var, tv)):
        ref = (t.double() * w.double()[:, None]).sum(0)
        check(got, ref, torch.float32, 1, 4 * U * (t.double().abs() * w.double()[:, None]).sum(0), what="merge_tiles")
    gamma, beta = _randn((C,), 4) * 0.3 + 1, _randn((C,), 5) * 0.3
    out = _Out(B * HW, C, dtype)
    ops.groupnorm_apply(x, B, HW, out.view, gamma, beta, 1e-6, True, mean=mean, var=var)
    y = out.done("GN apply (explicit statistics)")
    z = torch.zeros(B, 32, dtype=torch.float64, device="cuda")
    ref, err = _gn_expected(x, B, HW, C, mean.double().view(B, 32), var.double().view(B, 32), z, z, gamma, beta, 1e-6, True)
    check(y, ref, dtype, 1, err, frac=FRAC["groupnorm"][dtype == torch.float16], what=f"GN explicit stats C={C} {dt}")
    ms, vs = torch.empty(B * 32), torch.empty(B * 32)
    cpu_ops.groupnorm_merge_tiles(*_cpu(tm, tv, w), ms, vs)
    for got, t in ((ms, tm), (vs, tv)):
        ref_t = (t.double() * w.double()[:, None]).sum(0)
        check(got.cuda(), ref_t, torch.float32, 1, 4 * U * (t.double().abs() * w.double()[:, None]).sum(0), what="stand-in merge_tiles")
    ys = cpu_ops.groupnorm_apply(*_cpu(x), B, HW, torch.empty(B * HW, C, dtype=dtype), *_cpu(gamma, beta), 1e-6, True, mean=mean.cpu(),
                                 var=var.cpu())
    check(ys.cuda(), ref, dtype, 1, err, frac=FRAC["groupnorm"][dtype == torch.float16], what=f"stand-in GN explicit stats C={C} {dt}")


@pytest.mark.gpu
@pytest.mark.parametrize("dt", list(DT))
@pytest.mark.parametrize("C,C1,cs", [(320, 320, 0.7), (320, 168, 0.7), (640, 320, 1.0), (320, 168, 0.0)])
def test_zerosft_vs_fp64(C, C1, cs, dt):
    """out = lerp(h_raw, GN(h) * E(gamma + 1) + beta, cs); C1 = C (no skip), C1 inside a group (cpg 10), ldgb != 2C; at
    control_scale 0 the output is h_raw bit for bit."""
    ops, _ = _ops()
    dtype, B, HW = DT[dt], 2, 1500
    h = _gn_input(B, HW, C, dtype, 40 + C1)
    skip = _strided(_randn((B * HW, C - C1), 41, dtype=dtype), 16) if C1 < C else None
    gb = _randn((B * HW, 2 * C + 24), 42, 0.3, dtype)[:, 8:8 + 2 * C]
    gw, gbias = _randn((C,), 43) * 0.3 + 1, _randn((C,), 44) * 0.3
    sums = torch.zeros(ops.groupnorm_ws_size(B, HW, C), dtype=torch.float64, device="cuda")
    ops.groupnorm_stats(h, B, HW, sums)
    out = _Out(B * HW, C, dtype)
    ops.zerosft_apply(h, skip, C1, gb, out.view, B, HW, sums, gw, gbias, 1e-5, torch.tensor([cs], device="cuda"))
    y = out.done("ZeroSFT")
    raw = h if skip is None else torch.cat([h[:, :C1], skip], 1)
    if cs == 0.0:
        assert torch.equal(y, raw), "control_scale 0 must return h_raw bit for bit"
        return
    kp, ppb, _ = _gn_stats_shape(HW, C)
    _, _, _, m, v, dm, dv = _gn_reference(h, B, HW, C, ppb // kp + kp + 4)
    n, nerr = _gn_expected(h, B, HW, C, m, v, dm, dv, gw, gbias, 1e-5, False)
    g1 = (gb[:, :C].float() + 1).to(dtype).double()
    bb = gb[:, C:].double()
    csf = torch.tensor(cs, dtype=torch.float32)
    ref = (n * g1 + bb) * float(csf) + raw.double() * float(1 - csf)
    err = (nerr * g1.abs() + 8 * U * ((n * g1).abs() + bb.abs())) * cs + 4 * U * raw.double().abs()
    check(y, ref, dtype, 1, err, frac=FRAC["groupnorm"][dtype == torch.float16], what=f"ZeroSFT C={C} C1={C1} {dt}")
    hc = h.cpu()
    ws = cpu_ops.groupnorm_stats(hc, B, HW, torch.zeros(cpu_ops.groupnorm_ws_size(B, HW, C), dtype=torch.float64))
    ys = cpu_ops.zerosft_apply(hc, *_cpu(skip, C1, gb), torch.empty(B * HW, C, dtype=dtype), B, HW, ws, *_cpu(gw, gbias), 1e-5,
                               torch.tensor([cs]))
    check(ys.cuda(), ref, dtype, 1, err, frac=FRAC["groupnorm"][dtype == torch.float16], what=f"stand-in ZeroSFT C={C} C1={C1} {dt}")


# ------------------------------------------------------------------------------------------------------------------
# LayerNorm (all three register-tile instantiations, several rows per warp), row softmax (both kernels)
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dt", list(DT))
@pytest.mark.parametrize("rows", ["1", "300", "walk"])
@pytest.mark.parametrize("C", [320, 768, 776, 1280, 1288, 2048])
def test_layernorm_and_stats_vs_fp64(C, rows, dt):
    """C covers MAXV 3 / 5 / 8 and both sides of each limit; 'walk' = 3 * SMs * 16 * 8 + 5 rows makes every warp walk
    several rows, through the next-row prefetch."""
    ops, _ = _ops()
    dtype = DT[dt]
    R = {"1": 1, "300": 300, "walk": 3 * _sms() * 16 * 8 + 5}[rows]
    x = _strided((_randn((R, C), 60) * 1.5 + 0.3 * _randn((R, 1), 61)).to(dtype), 8)
    gamma, beta = _randn((C,), 62) * 0.3 + 1, _randn((C,), 63) * 0.3
    out = _Out(R, C, dtype)
    ops.layernorm(x, out.view, gamma, beta)
    y = out.done(f"LayerNorm C={C}")
    xd = x.double()
    m = xd.mean(1, keepdim=True)
    rstd = 1 / torch.sqrt(xd.var(1, unbiased=False, keepdim=True) + 1e-5)
    cl = C // 32 + 16                               # per-lane sequential adds + the warp tree
    dm = cl * U * xd.abs().mean(1, keepdim=True)
    ref = (xd - m) * rstd * gamma.double() + beta.double()
    err = gamma.double().abs() * rstd * ((xd - m).abs() * (cl + 8) * U + dm) + 8 * U * ((xd - m).abs() * rstd * gamma.double().abs() + beta.double().abs())
    check(y, ref, dtype, 1, err, frac=FRAC["layernorm"][dtype == torch.float16], what=f"LayerNorm C={C} rows={R} {dt}")
    stats = torch.full((R, 2), math.nan, device="cuda")
    ops.layernorm_stats(x, stats)
    check(stats[:, 0], rstd[:, 0], torch.float32, 1, (cl + 8) * U * rstd[:, 0], what="LN stats rstd")
    check(stats[:, 1], (m * rstd)[:, 0], torch.float32, 1, ((cl + 8) * U * m.abs() + dm)[:, 0] * rstd[:, 0], what="LN stats mean*rstd")
    if rows != "walk":                              # the stand-ins on the CPU: one row count is enough
        xc = x.cpu()
        ys = cpu_ops.layernorm(xc, torch.empty(R, C, dtype=dtype), *_cpu(gamma, beta))
        check(ys.cuda(), ref, dtype, 1, err, frac=FRAC["layernorm"][dtype == torch.float16], what=f"stand-in LayerNorm C={C} {dt}")
        st = cpu_ops.layernorm_stats(xc, torch.empty(R, 2)).cuda()
        check(st[:, 0], rstd[:, 0], torch.float32, 1, (cl + 8) * U * rstd[:, 0], what="stand-in LN stats rstd")
        check(st[:, 1], (m * rstd)[:, 0], torch.float32, 1, ((cl + 8) * U * m.abs() + dm)[:, 0] * rstd[:, 0], what="stand-in LN stats mean*rstd")


def _softmax_rows_input(rows, cols, seed):
    S = _randn((rows, cols), seed, 16.0)           # * scale 0.25 -> logits ~ N(0, 4): a few keys carry most of the mass
    S[1] = 1e4                                      # all equal and large: uniform
    S[2, :] = -50.0
    S[2, 7], S[2, cols - 1] = 88.0, 88.0            # two equal maxima
    S[3, ::3] = 3e3                                 # a third of the row tied at the maximum
    return S


@pytest.mark.gpu
@pytest.mark.parametrize("aligned", [True, False])
@pytest.mark.parametrize("cols", [1000, 1023, 1024, 4097, 18496])
def test_softmax_rows_vs_fp64(cols, aligned):
    """cols >= 1024 with aligned operands take the shared-memory kernel; an odd output offset forces the generic one."""
    ops, _ = _ops()
    rows, scale = 40, 0.25
    S = _strided(_randn((rows, cols), 1), 4 + (-cols) % 4).copy_(_softmax_rows_input(rows, cols, 70))
    out = _Out(rows, cols, torch.bfloat16, lo=None if aligned else 1)
    ops.softmax_rows(S, out.view, cols, scale)
    P = out.done(f"softmax cols={cols}")
    Sd = S.double()
    z = (Sd - Sd.max(1, keepdim=True).values) * scale
    e = torch.exp(z)
    ref = e / e.sum(1, keepdim=True)
    err = ref * U * (3 * z.abs() + cols / 256 + 32)
    check(P, ref, torch.bfloat16, 1, err, frac=FRAC["softmax"][0], what=f"softmax cols={cols} aligned={aligned}")


# ------------------------------------------------------------------------------------------------------------------
# entry / exit convolutions
# ------------------------------------------------------------------------------------------------------------------
def _conv_ref(x, w, bias):
    """fp64 conv (padding 1) and the matching sum of magnitudes."""
    y = F.conv2d(x.double(), w.double(), None if bias is None else bias.double(), padding=1)
    mag = F.conv2d(x.double().abs(), w.double().abs(), None if bias is None else bias.double().abs(), padding=1)
    return y, mag


def _nhwc(t):
    B, C, H, W = t.shape
    return t.permute(0, 2, 3, 1).reshape(B * H * W, C)


SMALL_CIN_SHAPES = [(2, 37, 45), (1, 1, 67), (3, 29, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("dt", list(DT))
@pytest.mark.parametrize("Cout", [8, 320, 512])
@pytest.mark.parametrize("Cin", list(range(1, 9)))
def test_conv3x3_small_cin_vs_fp64(Cin, Cout, dt):
    """Strided NCHW tile views (B > 1, H or W = 1), > 48 KB of shared-memory weights at Cout 512, a residual with
    ldr != Cout; the accumulator is rounded to E before the residual is added. im2col_3x3_small_cin equals F.unfold exactly."""
    ops, _ = _ops()
    dtype = DT[dt]
    w = _randn((Cout, Cin, 3, 3), 80, 0.3)
    bias = _randn((Cout,), 81, 0.2)
    for i, (B, H, W) in enumerate(SMALL_CIN_SHAPES):
        big = _randn((B, Cin + 1, H + 5, W + 7), 82 + i, 2.0)
        x = big[:, 1:, 2:2 + H, 3:3 + W]
        xe = x.to(dtype).double()
        res = _strided(_randn((B * H * W, Cout), 85 + i, dtype=dtype), 24) if i != 1 else None
        out = _Out(B * H * W, Cout, dtype)
        ops.conv3x3_small_cin(x, w, bias, out.view, residual=res)
        y = out.done(f"small_cin Cin={Cin} Cout={Cout}")
        acc, mag = _conv_ref(xe, w, bias)
        acc, mag = _nhwc(acc), _nhwc(mag)
        err = (9 * Cin + 1) * U * mag
        ys = cpu_ops.conv3x3_small_cin(*_cpu(x, w, bias), torch.empty(B * H * W, Cout, dtype=dtype), residual=_cpu(res)[0]).cuda()
        for who, got in (("", y), ("stand-in ", ys)):
            if res is None:
                check(got, acc, dtype, 1, err, frac=FRAC["small_cin"][dtype == torch.float16], what=f"{who}small_cin {Cin}->{Cout} {B}x{H}x{W} {dt}")
            else:
                ref = acc.to(dtype).double() + res.double()
                check(got, ref, dtype, 1, err + ulp(acc, dtype), frac=FRAC["small_cin_res"][dtype == torch.float16],
                      what=f"{who}small_cin+res {Cin}->{Cout} {B}x{H}x{W} {dt}")
        KP = (Cin * 9 + 63) // 64 * 64
        cols = _Out(B * H * W, KP, dtype)
        from supir_b200 import _native
        name = "supir_im2col_3x3_small_cin" if dtype == torch.bfloat16 else "supir_im2col_3x3_small_cin_f16"
        _native.call(name, ops._ptr(x), x.stride(0), x.stride(1), x.stride(2), ops._ptr(cols.view), cols.view.stride(0),
                     B, H, W, Cin, KP, ops._stream())
        got = cols.done("im2col_small_cin")
        ref = torch.zeros(B * H * W, KP, dtype=dtype, device="cuda")
        ref[:, :Cin * 9] = F.unfold(x, 3, padding=1).permute(0, 2, 1).reshape(B * H * W, Cin * 9).to(dtype)
        assert torch.equal(got, ref), f"im2col_small_cin Cin={Cin} {B}x{H}x{W}"


@pytest.mark.gpu
@pytest.mark.parametrize("dt", list(DT))
@pytest.mark.parametrize("Cout", [3, 4, 8])
@pytest.mark.parametrize("Cin", [64, 320, 512])
def test_conv3x3_small_cout_vs_fp64(Cin, Cout, dt):
    """Crop windows touching each border, written into an offset canvas (ob != C*h*w); Cin > 256 takes the lane loop's
    second pass over channel vectors."""
    ops, _ = _ops()
    dtype, B, H, W = DT[dt], 2, 23, 31
    x = _randn((B, Cin, H, W), 90, dtype=dtype)
    w = (_randn((Cout, Cin, 3, 3), 91) / math.sqrt(9 * Cin))
    bias = _randn((Cout,), 92, 0.2)
    xt = _strided(_nhwc(x), 8)
    acc, mag = _conv_ref(x, w, bias)
    cn = 9 * 8 * (-(-Cin // 256)) + 16
    for y0, x0, ch, cw in [(0, 0, H, W), (0, 9, 11, W - 9), (5, 0, H - 5, 13), (H - 1, W - 1, 1, 1)]:
        can = _Canvas(B, Cout, ch, cw)
        ops.conv3x3_small_cout(xt, B, H, W, w.permute(0, 2, 3, 1).contiguous(), bias, can.view, crop=(y0, x0, ch, cw))
        got = can.done(f"small_cout crop {(y0, x0, ch, cw)}")
        sl = (slice(None), slice(None), slice(y0, y0 + ch), slice(x0, x0 + cw))
        check(got, acc[sl], dtype, 1, cn * U * mag[sl], frac=FRAC["small_cout"][dtype == torch.float16], what=f"small_cout {Cin}->{Cout} crop {(y0, x0, ch, cw)} {dt}")
        ys = cpu_ops.conv3x3_small_cout(*_cpu(xt), B, H, W, *_cpu(w.permute(0, 2, 3, 1).contiguous(), bias), torch.empty(B, Cout, ch, cw),
                                        crop=(y0, x0, ch, cw)).cuda()
        check(ys, acc[sl], dtype, 1, cn * U * mag[sl], frac=FRAC["small_cout"][dtype == torch.float16], what=f"stand-in small_cout {Cin}->{Cout} {dt}")


@pytest.mark.gpu
def test_conv1x1_small_nchw_vs_fp64():
    ops, _ = _ops()
    B, H, W = 2, 19, 23
    for cin in range(1, 9):
        x = _randn((B, cin, H, W), 100 + cin, 3.0)
        xin = (x * 0.18215).to(torch.bfloat16).double()           # in_scale, then rounded to bf16 in fp32
        for cout in range(1, 9):
            w, b = _randn((cout, cin), 110 + cout, 0.5), _randn((cout,), 120 + cout, 0.2)
            y = _Flat((B, cout, H, W), torch.float32)
            ops.conv1x1_small_nchw(x, w, b, y.view, in_scale=0.18215)
            got = y.done(f"conv1x1 {cin}->{cout}")
            ref = torch.einsum("bchw,oc->bohw", xin, w.double()) + b.double()[:, None, None]
            mag = torch.einsum("bchw,oc->bohw", xin.abs(), w.double().abs()) + b.double().abs()[:, None, None]
            check(got, ref, torch.bfloat16, 1, (cin + 2) * U * mag, frac=FRAC["conv1x1"][0], what=f"conv1x1 {cin}->{cout}")
            ys = cpu_ops.conv1x1_small_nchw(*_cpu(x, w, b), torch.empty(B, cout, H, W), in_scale=0.18215).cuda()
            check(ys, ref, torch.bfloat16, 1, (cin + 2) * U * mag, frac=FRAC["conv1x1"][0], what=f"stand-in conv1x1 {cin}->{cout}")


# ------------------------------------------------------------------------------------------------------------------
# exact kernels, at sizes that wrap the grid-stride loops (SMs * 32 blocks * 256 threads items)
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_layout_kernels_exact_past_grid_stride_wrap():
    ops, _ = _ops()
    bf = torch.bfloat16
    B, H, W, C = 2, 64, 96, 320                     # upsample: 2 * 4 * 6144 * 40 = 1.97 M 16-byte items
    x4 = _randn((B, C, H, W), 130, dtype=bf)
    xt = _strided(_nhwc(x4), 8)
    up = _Out(B * 4 * H * W, C, bf)
    ops.upsample2x(xt, B, H, W, up.view)
    ref = _nhwc(F.interpolate(x4.float(), scale_factor=2, mode="nearest")).to(bf)
    assert torch.equal(up.done("upsample2x"), ref)
    xc = xt.cpu()
    assert torch.equal(cpu_ops.upsample2x(xc, B, H, W, torch.empty(B * 4 * H * W, C, dtype=bf)), ref.cpu()), "stand-in upsample2x"
    for pad_lo in (1, 0):
        Ho, Wo = ((H - 1) // 2 + 1, (W - 1) // 2 + 1) if pad_lo else ((H - 2) // 2 + 1, (W - 2) // 2 + 1)
        cols = _Flat((B * Ho * Wo, 9 * C), bf)
        ops.im2col_s2(xt, B, H, W, cols.view, Ho, Wo, pad_lo)
        xp = F.pad(x4.float(), (1, 1, 1, 1) if pad_lo else (0, 1, 0, 1))
        ref = F.unfold(xp, 3, stride=2).view(B, C, 9, Ho * Wo).permute(0, 3, 2, 1).reshape(B * Ho * Wo, 9 * C).to(bf)
        assert torch.equal(cols.done(f"im2col_s2 pad_lo={pad_lo}"), ref)
        assert torch.equal(cpu_ops.im2col_s2(xc, B, H, W, torch.empty(B * Ho * Wo, 9 * C, dtype=bf), Ho, Wo, pad_lo), ref.cpu()), \
            "stand-in im2col_s2"
    dst = _Out(B * H * W, C, bf)
    ops.copy2d(xt, dst.view)
    assert torch.equal(dst.done("copy2d"), xt)
    assert torch.equal(cpu_ops.copy2d(xc, torch.empty(B * H * W, C, dtype=bf)), xc), "stand-in copy2d"
    xf = _randn((B, C, H, W), 131)
    o = _Out(B * H * W, C, bf)
    ops.nchw_f32_to_nhwc_bf16(xf, o.view)
    assert torch.equal(o.done("nchw->nhwc"), _nhwc(xf).to(bf))
    back = _Flat((B, C, H, W), torch.float32)
    ops.nhwc_bf16_to_nchw_f32(xt, B, C, H * W, back.view)
    assert torch.equal(back.done("nhwc->nchw"), x4.float())


@pytest.mark.gpu
@pytest.mark.parametrize("dt", list(DT))
def test_crop_exit_exact(dt):
    from supir_b200 import _native
    ops, _ = _ops()
    dtype, B, H, W, C = DT[dt], 2, 150, 160, 8      # 2 * 8 * 140 * 150 = 336 k items; two windows on the image edges
    x = _strided(_randn((B * H * W, C), 140, dtype=dtype), 8)
    x4 = x.float().reshape(B, H, W, C).permute(0, 3, 1, 2)
    for y0, x0, ch, cw in [(0, 0, 140, 150), (10, 10, 140, 150), (0, 159, 150, 1)]:
        can = _Canvas(B, C, ch, cw)
        name = "supir_nhwc_bf16_crop_to_nchw_f32" if dtype == torch.bfloat16 else "supir_nhwc_f16_crop_to_nchw_f32"
        v = can.view
        _native.call(name, ops._ptr(x), x.stride(0), ops._ptr(v), v.stride(0), v.stride(1), v.stride(2), B, H, W, C, y0, x0, ch, cw,
                     ops._stream())
        assert torch.equal(can.done("crop exit"), x4[:, :, y0:y0 + ch, x0:x0 + cw])


@pytest.mark.gpu
@pytest.mark.parametrize("dt", list(DT))
def test_f32_to_16_and_axpy_exact(dt):
    ops, _ = _ops()
    dtype = DT[dt]
    n = 3_000_003
    x = _randn((n,), 150, 10.0)
    b = torch.tensor([1 + 2 ** -8, 1 + 3 * 2 ** -8, -(1 + 2 ** -8), 1 + 2 ** -11, 1 + 3 * 2 ** -11, math.inf, -math.inf, math.nan,
                      1e-40, -3e-39, 6e-8, 3e-8, 2.9e-8, 1e-9, 65504.0, 65519.0, 65520.0, 7e4, -1e5, 3.4e38, 0.0, -0.0],
                     device="cuda")
    x[:b.numel()] = b
    x[n // 2:n // 2 + b.numel()] = b
    x[-b.numel():] = b
    y = _Flat((n,), dtype)
    (ops.f32_to_bf16 if dtype == torch.bfloat16 else ops.f32_to_f16)(x, y.view)
    torch.cuda.synchronize()
    assert y.borders_ok(), "f32_to_16 wrote outside its output"
    got, ref = y.view, x.to(dtype)
    keep = ~torch.isnan(ref)
    assert torch.equal(torch.isnan(got), ~keep), "NaN inputs must give NaN, and only they (unwritten elements stay NaN)"
    assert torch.equal(got.view(torch.int16)[keep], ref.view(torch.int16)[keep]), "f32 -> 16-bit differs from torch's cast"
    if dtype == torch.bfloat16:
        ys = cpu_ops.f32_to_bf16(x.cpu(), torch.empty(n, dtype=dtype)).cuda()
        assert torch.equal(ys.view(torch.int16)[keep], ref.view(torch.int16)[keep]), "stand-in f32_to_bf16"
    rows, cols = 9000, 320                           # 360 k 16-byte items
    a = _strided(_randn((rows, cols), 151, dtype=dtype), 16)
    yy = _strided(_randn((rows, cols), 152, 3.0, dtype), 8)
    s = torch.tensor([0.7], device="cuda")
    out = _Out(rows, cols, dtype)
    ops.axpy(a, yy, out.view, s)
    ref = (a.float() + (yy.float() * s).to(dtype).float()).to(dtype)
    assert torch.equal(out.done("axpy"), ref)
    assert torch.equal(cpu_ops.axpy(*_cpu(a, yy), torch.empty(rows, cols, dtype=dtype), s.cpu()).cuda(), ref), "stand-in axpy"


# ------------------------------------------------------------------------------------------------------------------
# embeddings, small-batch Linear
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dim", [320, 1280])
def test_timestep_embedding_vs_fp64(dim):
    """Bound from fp32 argument rounding: the frequency exp(-ln(1e4) k / half) and the product t * f carry a relative error
    of about (3 |ln(1e4) k / half| + 5) * 2^-24, which sin / cos turn into an absolute error of |t f| times that."""
    ops, _ = _ops()
    t = torch.tensor([0.0, 0.37, 13.0, 401.5, 999.0], device="cuda")
    y = _Flat((5, dim), torch.float32)
    ops.timestep_embedding(t, y.view)
    got = y.done("timestep_embedding")
    half = dim // 2
    k = torch.arange(half, dtype=torch.float64, device="cuda")
    ex = math.log(10000.0) * k / half
    arg = t.double()[:, None] * torch.exp(-ex)[None]
    ref = torch.cat([torch.cos(arg), torch.sin(arg)], 1)
    darg = arg.abs() * U * (3 * ex + 5)[None]
    err = torch.cat([darg, darg], 1) + 4 * U
    assert bool(((got.double() - ref).abs() <= err).all()), float((got.double() - ref).abs().max())
    assert float(err.max()) < 1.3e-3
    ys = cpu_ops.timestep_embedding(t.cpu(), torch.empty(5, dim)).cuda()
    assert bool(((ys.double() - ref).abs() <= err).all()), f"stand-in: {float((ys.double() - ref).abs().max())}"


@pytest.mark.gpu
@pytest.mark.parametrize("dt", list(DT))
@pytest.mark.parametrize("K", [320, 1280, 2816])
@pytest.mark.parametrize("B", [1, 4, 5, 16])
def test_linear_small_m_vs_fp64(B, K, dt):
    """Every silu_in / silu_out / add combination; N = 1283 (not a multiple of 8); ldx, ldy, ldadd larger than the widths.
    Rounding points: the input (and its SiLU), the Linear output, the SiLU, the sum with `add`, the SiLU of the sum."""
    ops, _ = _ops()
    dtype, N = DT[dt], 1283
    x = _strided(_randn((B, K), 160, 2.0), 8)
    w = _randn((N, K), 161, 1 / math.sqrt(K), dtype)
    bias = _randn((N,), 162, 0.2)
    add = _strided(_randn((B, N), 163), 5)
    wd = w.double()
    for silu_in in (0, 1):
        xr = x.to(dtype).double()
        if silu_in:
            xr = F.silu(xr.float()).to(dtype).double()
        in_err = (ulp(xr, dtype) @ wd.abs().t()) if silu_in else 0.0     # the E-rounding of SiLU(x) may flip by one ulp
        acc = xr @ wd.t() + bias.double()
        err = (K / 32 + 16) * U * (xr.abs() @ wd.abs().t() + bias.double().abs()) + in_err
        for silu_out in range(4):
            for with_add in (False, True):
                v = acc.to(dtype).double()
                tol = ulp(acc, dtype) + err
                if silu_out & 1:
                    s = _silu64(v)
                    v, tol = s.to(dtype).double(), ulp(s, dtype) + 1.1 * tol + 8 * U * s.abs()
                if with_add:
                    s = v + add.double()
                    v, tol = s.to(dtype).double(), ulp(s, dtype) + tol
                if silu_out & 2:
                    s = _silu64(v)
                    v, tol = s.to(dtype).double(), ulp(s, dtype) + 1.1 * tol + 8 * U * s.abs()
                out = _Out(B, N, torch.float32)
                ops.linear_small_m(x, w, bias, out.view, silu_in=bool(silu_in), silu_out=silu_out, add=add if with_add else None)
                got = out.done("linear_small_m")
                what = f"linear_small_m B={B} K={K} silu_in={silu_in} silu_out={silu_out} add={with_add} {dt}"
                frac = FRAC["linear_small_m"][dtype == torch.float16]
                check(got, v, dtype, 0, tol, frac=frac, what=what)
                assert torch.equal(got.to(dtype).float(), got), f"{what}: output is not rounded to {dt}"
                ys = cpu_ops.linear_small_m(*_cpu(x, w, bias), torch.empty(B, N), silu_in=bool(silu_in), silu_out=silu_out,
                                            add=add.cpu() if with_add else None).cuda()
                check(ys, v, dtype, 0, tol, frac=frac, what="stand-in " + what)


# ------------------------------------------------------------------------------------------------------------------
# attention variants
# ------------------------------------------------------------------------------------------------------------------
def _att_ref(q, k, v, B, H, Lq, Lk, D, scale):
    out = torch.empty(B * Lq, H * D, dtype=torch.float64, device="cuda")
    for b in range(B):
        qb = q[b * Lq:(b + 1) * Lq].double().view(Lq, H, D).transpose(0, 1)
        kb = k[b * Lk:(b + 1) * Lk].double().view(Lk, H, D).transpose(0, 1)
        vb = v[b * Lk:(b + 1) * Lk].double().view(Lk, H, D).transpose(0, 1)
        p = torch.softmax(qb @ kb.transpose(1, 2) * scale, -1)
        out[b * Lq:(b + 1) * Lq] = (p @ vb).transpose(0, 1).reshape(Lq, H * D)
    return out


def _set_att(lib, emu, pack):
    lib.supir_set_attention_exp_emulation(emu)
    lib.supir_set_attention_alu_pack(pack)


@pytest.mark.gpu
@pytest.mark.parametrize("emu", [0, 2, 4])
@pytest.mark.parametrize("L", [1, 63, 65, 300])
def test_attention_1head_512_exp_emulation(L, emu):
    from test_gpu_bench_shapes import _check_attention
    ops, lib = _ops()
    B, D = 2, 512
    qkv = _randn((B * L, 3 * D + 8), 170, 1.0, torch.bfloat16)
    q, k, v = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:3 * D]
    out = _Out(B * L, D, torch.bfloat16)
    try:
        _set_att(lib, emu, -1)
        ops.attention_1head(q, k, v, out.view, B, L)
    finally:
        _set_att(lib, -1, -1)
    ref = _att_ref(q, k, v, B, 1, L, L, D, D ** -0.5).float()
    _check_attention(out.done("1-head attention"), ref, f"1-head L={L} emu={emu}")
    if emu == 0:
        ys = cpu_ops.attention_1head(*_cpu(q, k, v), torch.empty(B * L, D, dtype=torch.bfloat16), B, L).cuda()
        _check_attention(ys, ref, f"stand-in 1-head L={L}")


@pytest.mark.gpu
@pytest.mark.parametrize("emu", [0, 2, 4])
def test_attention_1head_two_key_softmax_is_unbiased(emu):
    """Each query sees two keys with logits 0 and -d (d spread over (0, 4) log2 units) and every other key far below; value
    rows 0 and 1 are 0 and 1. So out = E(P1) / (1 + P1) with P1 = 2^x: the kernel's exponential (MUFU, or the FMA-pipe
    polynomial under exp_emulation) is seen directly. The mean relative error over 4096 queries must be far below what
    a 1e-3 error in the exponential's cubic coefficient would give (~1.5e-4), and the outputs must mostly be the correctly
    rounded model value."""
    ops, lib = _ops()
    L, D = 4096, 512
    scale = D ** -0.5
    q = torch.zeros(L, D, device="cuda")
    q[:, 1] = -torch.rand(L, generator=_gen(180), device="cuda") * 7.0          # logit of key 1 = q1 * 8 * scale
    q[:, 2] = 1.0
    k = torch.zeros(L, D, device="cuda")
    k[0, 0], k[1, 1] = 8.0, 8.0
    k[2:, 2] = -3e4                                                             # every other key: 2^-1900 -> 0
    v = torch.zeros(L, D, device="cuda")
    v[1] = 1.0
    q, k, v = (t.to(torch.bfloat16) for t in (q, k, v))
    out = _Out(L, D, torch.bfloat16)
    try:
        _set_att(lib, emu, -1)
        ops.attention_1head(q, k, v, out.view, 1, L)
    finally:
        _set_att(lib, -1, -1)
    got = out.done("two-key attention")[:, 0].double()
    sl2 = torch.tensor(scale, dtype=torch.float32) * torch.tensor(1.4426950408889634, dtype=torch.float32)
    x = (q[:, 1].float() * 8.0) * sl2                                           # fp32 logit in log2 units (max is 0)
    p1 = torch.exp2(x.double())
    ref = (p1.to(torch.bfloat16).double() / (1 + p1)).to(torch.bfloat16).double()
    rel = (got - ref) / ref
    bias = float(rel.mean())
    ne = float((got != ref).double().mean())
    print(f"two-key attention emu={emu}: mean rel err {bias:.3g}, {ne:.3g} differ from the model")
    assert abs(bias) <= 7e-5, f"emu={emu}: mean relative error {bias:.3g}"    # measured 0 / 2.3e-5 / 3.6e-5 at emu 0 / 2 / 4
    assert ne <= 0.04, f"emu={emu}: {ne:.3g} of the outputs differ from the correctly rounded model"


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(2, 3, 1, 77), (2, 3, 300, 1), (1, 5, 200, 333)])
def test_attention_h64_alu_pack_and_edges(shape):
    """ALU packing 1 and 3 (never the default) vs fp64 and vs the conversion-unit packing (they differ only on exact ties),
    with Lq = 1 and Lk = 1."""
    from test_gpu_bench_shapes import _check_attention
    ops, lib = _ops()
    B, H, Lq, Lk = shape
    C = H * 64
    q = _randn((B * Lq, C), 190, 1.5, torch.bfloat16)
    kv = _randn((B * Lk, 2 * C), 191, 1.5, torch.bfloat16)
    k, v = kv[:, :C].contiguous(), kv[:, C:].contiguous()
    ref = _att_ref(q, k, v, B, H, Lq, Lk, 64, 0.125).float()
    outs = {}
    try:
        for pack in (0, 1, 3):
            _set_att(lib, 0, pack)
            o = _Out(B * Lq, C, torch.bfloat16)
            ops.attention(q, k, v, o.view, B, H, Lq, Lk)
            outs[pack] = o.done(f"attention pack={pack}")
            _check_attention(outs[pack], ref, f"h64 {shape} alu_pack={pack}")
    finally:
        _set_att(lib, -1, -1)
    for pack in (1, 3):
        assert float((outs[pack] != outs[0]).double().mean()) <= 1e-2, f"alu_pack={pack} differs beyond ties"
    ys = cpu_ops.attention(*_cpu(q, k, v), torch.empty(B * Lq, C, dtype=torch.bfloat16), B, H, Lq, Lk).cuda()
    _check_attention(ys, ref, f"stand-in h64 {shape}")


@pytest.mark.gpu
def test_attention_h64_fused_qkv_slices():
    """q / k / v as column slices of one fused [M, 3C] projection (how the networks call it) give the bits of contiguous
    copies."""
    ops, _ = _ops()
    B, H, L = 2, 5, 333
    C = H * 64
    qkv = _randn((B * L, 3 * C), 195, 1.5, torch.bfloat16)
    o1, o2 = _Out(B * L, C, torch.bfloat16), _Out(B * L, C, torch.bfloat16)
    ops.attention(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], o1.view, B, H, L, L)
    ops.attention(qkv[:, :C].contiguous(), qkv[:, C:2 * C].contiguous(), qkv[:, 2 * C:].contiguous(), o2.view, B, H, L, L)
    assert torch.equal(o1.done("fused"), o2.done("contiguous"))


# ------------------------------------------------------------------------------------------------------------------
# text-tower kernels (fp32 residual stream, short causal attention, embedding gathers), sampler elementwise
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("L", [1, 127, 128])
def test_attention_small_vs_fp64(L):
    """L up to the kernel's 128-token limit, leading dimensions > H * 64, causal and not. Everything is fp32 up to the bf16
    output: per row, each probability carries (128 * sum|q k| * scale + 3 |logit - max| + 4) * 2^-24 of relative error."""
    ops, _ = _ops()
    bf, B, H = torch.bfloat16, 3, 4
    C = H * 64
    q, k, v = (_strided(_randn((B * L, C), 300 + i, 1.5, bf), 8 * (i + 1)) for i in range(3))
    qd, kd, vd = (t.double().view(B, L, H, 64).transpose(1, 2) for t in (q, k, v))
    s_ = qd @ kd.transpose(-1, -2) * 0.125
    dot = qd.abs() @ kd.abs().transpose(-1, -2) * 0.125
    for causal in (True, False):
        allowed = torch.ones(L, L, dtype=torch.bool, device="cuda")
        if causal:
            allowed = torch.tril(allowed)
        sm = s_.masked_fill(~allowed, -math.inf)
        p = torch.softmax(sm, -1)
        z = (sm - sm.max(-1, keepdim=True).values).masked_fill(~allowed, 0).abs()
        rel = ((128 * dot + 3 * z).masked_fill(~allowed, 0).amax(-1, keepdim=True) + L + 8) * U
        ref = (p @ vd).transpose(1, 2).reshape(B * L, C)
        err = (rel * (p @ vd.abs())).transpose(1, 2).reshape(B * L, C)
        out = _Out(B * L, C, bf)
        ops.attention_small(q, k, v, out.view, B, H, L, causal=causal)
        check(out.done("attention_small"), ref, bf, 1, err, frac=FRAC["attention_small"][0], what=f"attention_small L={L} causal={causal}")
        ys = cpu_ops.attention_small(*_cpu(q, k, v), torch.empty(B * L, C, dtype=bf), B, H, L, causal=causal).cuda()
        check(ys, ref, bf, 1, err, frac=FRAC["attention_small"][0], what=f"stand-in attention_small L={L} causal={causal}")


@pytest.mark.gpu
@pytest.mark.parametrize("outputs", ["bf16", "f32", "both"])
def test_layernorm_f32_vs_fp64(outputs):
    """fp32 rows (ld > C), enough of them that warps walk several rows; either output may be absent."""
    ops, _ = _ops()
    R, C = 3 * _sms() * 8 * 8 + 5, 1280
    x = _strided(_randn((R, C), 310, 1.5) + _randn((R, 1), 311), 4)
    gamma, beta = _randn((C,), 312) * 0.3 + 1, _randn((C,), 313) * 0.3
    ob = _Out(R, C, torch.bfloat16) if outputs != "f32" else None
    of = _Out(R, C, torch.float32) if outputs != "bf16" else None
    ops.layernorm_f32(x, gamma, beta, out_bf16=None if ob is None else ob.view, out_f32=None if of is None else of.view)
    xd = x.double()
    m = xd.mean(1, keepdim=True)
    rstd = 1 / torch.sqrt(xd.var(1, unbiased=False, keepdim=True) + 1e-5)
    cl = C // 32 + 16
    g, b = gamma.double(), beta.double()
    ref = (xd - m) * rstd * g + b
    err = g.abs() * rstd * ((xd - m).abs() * (cl + 8) * U + cl * U * xd.abs().mean(1, keepdim=True)) + \
        8 * U * ((xd - m).abs() * rstd * g.abs() + b.abs())
    sb = cpu_ops.layernorm_f32(*_cpu(x, gamma, beta), out_bf16=torch.empty(R, C, dtype=torch.bfloat16))
    sf = cpu_ops.layernorm_f32(*_cpu(x, gamma, beta), out_f32=torch.empty(R, C))
    if ob is not None:
        check(ob.done("layernorm_f32 bf16"), ref, torch.bfloat16, 1, err, frac=FRAC["layernorm"][0], what="layernorm_f32 -> bf16")
        check(sb.cuda(), ref, torch.bfloat16, 1, err, frac=FRAC["layernorm"][0], what="stand-in layernorm_f32 -> bf16")
    if of is not None:
        check(of.done("layernorm_f32 f32"), ref, torch.float32, 0, err, what="layernorm_f32 -> fp32")
        check(sf.cuda(), ref, torch.float32, 0, err, what="stand-in layernorm_f32 -> fp32")


@pytest.mark.gpu
def test_gather_rows_f32_exact_with_clamped_indices():
    """rows * C / 4 = 640 k items wrap the text kernels' grid-stride loop (SMs * 16 * 256); indices below 0 and past the table
    are clamped; with and without the positional rows (r % L)."""
    ops, _ = _ops()
    T, C, rows, L = 500, 1280, 2000, 77
    table = _strided(_randn((T, C), 320), 4)
    pos = _strided(_randn((L, C), 321), 8)
    idx = torch.randint(-40, T + 40, (rows,), generator=_gen(322), device="cuda", dtype=torch.int32)
    idx[:4] = torch.tensor([-1, 0, T - 1, T], dtype=torch.int32)
    base = table[idx.long().clamp(0, T - 1)]
    for p_ in (None, pos):
        out = _Out(rows, C, torch.float32)
        ops.gather_rows_f32(table, idx, out.view, pos=p_, L=L if p_ is not None else 0)
        ref = base if p_ is None else base + pos[torch.arange(rows, device="cuda") % L]
        assert torch.equal(out.done("gather_rows_f32"), ref), f"gather_rows_f32 pos={p_ is not None}"
        ys = cpu_ops.gather_rows_f32(*_cpu(table, idx), torch.empty(rows, C), pos=_cpu(p_)[0], L=L if p_ is not None else 0)
        assert torch.equal(ys.cuda(), ref), "stand-in gather_rows_f32"


@pytest.mark.gpu
def test_edm_pre_post_with_null_operands_vs_fp64():
    """eps, x_center and denoised each NULL; 2 x 4 x 400 x 400 elements wrap the grid-stride loop. A few fp32 operations per
    element: 16 * 2^-24 * (sum of the magnitudes) bounds each result."""
    ops, _ = _ops()
    shape = (2, 4, 400, 400)
    x, eps, xc = _randn(shape, 330), _randn(shape, 331), _randn(shape, 332)
    net = _randn((4,) + shape[1:], 333)
    nm, cin, cout, cfg, rmul, sig, dt_ = 0.37, 0.21, -3.1, 2.5, 0.4, 3.3, -0.9
    for e in (eps, None):
        xh, ni = _Flat(shape, torch.float32), _Flat((4,) + shape[1:], torch.float32)
        ops.edm_pre(x, e, nm, cin, xh.view, ni.view)
        xhd = x.double() + (0 if e is None else e.double() * nm)
        mag = x.double().abs() + (0 if e is None else (e.double() * nm).abs())
        check(xh.done("edm_pre x_hat"), xhd, torch.float32, 0, 4 * U * mag, what="edm_pre x_hat")
        check(ni.done("edm_pre net_in"), torch.cat([xhd * cin] * 2), torch.float32, 0, torch.cat([6 * U * mag * cin] * 2), what="edm_pre net_in")
        sx, sn = torch.empty(shape), torch.empty((4,) + shape[1:])
        cpu_ops.edm_pre(*_cpu(x, e), nm, cin, sx, sn)
        check(sx.cuda(), xhd, torch.float32, 0, 4 * U * mag, what="stand-in edm_pre")
    xh = x
    n = net.double().view(2, -1)
    du, dc = n[0] * cout + xh.double().view(-1), n[1] * cout + xh.double().view(-1)
    mden = (n.abs().sum(0) * abs(cout) + xh.double().abs().view(-1)) * (1 + 2 * abs(cfg))
    for center, want_den in ((xc, True), (None, True), (xc, False)):
        den = du + cfg * (dc - du)
        md = mden
        if center is not None:
            den = den - (den - center.double().view(-1)) * rmul
            md = mden * (1 + 2 * abs(rmul)) + center.double().abs().view(-1) * abs(rmul)
        xn = xh.double().view(-1) + (xh.double().view(-1) - den) / sig * dt_
        mx = xh.double().abs().view(-1) + (xh.double().abs().view(-1) + md) * abs(dt_ / sig)
        o, d = _Flat(shape, torch.float32), (_Flat(shape, torch.float32) if want_den else None)
        ops.edm_post(xh, net, center, cout, cfg, rmul, sig, dt_, o.view, None if d is None else d.view)
        what = f"edm_post x_center={center is not None} denoised={want_den}"
        check(o.done(what).view(-1), xn, torch.float32, 0, 16 * U * mx, what=what)
        if d is not None:
            check(d.done(what).view(-1), den, torch.float32, 0, 16 * U * md, what=what + " (denoised)")
        so = torch.empty(shape)
        cpu_ops.edm_post(*_cpu(xh, net, center), cout, cfg, rmul, sig, dt_, so)
        check(so.cuda().view(-1), xn, torch.float32, 0, 16 * U * mx, what="stand-in " + what)


@pytest.mark.gpu
def test_tile_gather_exact_on_image_edges():
    """Windows at every image edge and corner of a 2 x 4 x 150 x 170 latent; 9 windows of 128 x 128 wrap the grid-stride loop."""
    ops, _ = _ops()
    N, C, H, W, T = 2, 4, 150, 170, 128
    src = _randn((N, C, H, W), 340)
    wins = [(y, y + T, x, x + T) for y in (0, 11, H - T) for x in (0, 23, W - T)]
    table = torch.tensor(wins, dtype=torch.int32, device="cuda")
    out = _Flat((len(wins), N, C, T, T), torch.float32)
    ops.tile_gather(src, table, T, out.view)
    got = out.done("tile_gather")
    ref = torch.stack([src[:, :, a:b, c:d] for a, b, c, d in wins])
    assert torch.equal(got, ref)
    ys = cpu_ops.tile_gather(*_cpu(src, table), T, torch.empty(len(wins), N, C, T, T))
    assert torch.equal(ys.cuda(), ref), "stand-in tile_gather"


# ------------------------------------------------------------------------------------------------------------------
# bit-invariance: tile widths, batch sub-ranges
# ------------------------------------------------------------------------------------------------------------------
WIDTHS = (64, 128, 160, 256)


def _at_width(lib, bn, fn):
    lib.supir_set_gemm_tile_n(bn)
    try:
        return fn()
    finally:
        lib.supir_set_gemm_tile_n(0)


def _gemm_operands(name, dtype, M, K=320):
    from test_gpu_gemm_staged import EPILOGUES
    e = EPILOGUES[name]
    act = e.get("act", 0)
    N = 640 if act == 2 else 608
    a, w = _randn((M, K), 201, dtype=dtype), _randn((N, K), 202, 1 / math.sqrt(K), dtype)
    n_out = N // 2 if act == 2 else N
    kw = dict(act=act, bias=_randn((N,), 203, 0.2) if e.get("bias") else None)
    if e.get("rowvec"):
        kw.update(rowvec=_randn((M // 300 + 1, N), 204, 0.5), rows_per_batch=300)
    if e.get("ln"):
        kw["ln"] = (torch.stack([_randn((M,), 205).abs() + 0.5, _randn((M,), 206, 0.3)], 1).contiguous(), _randn((N,), 207, 0.5))
    if e.get("res"):
        kw["residual"] = _randn((M, n_out + 24), 208, dtype=dtype)[:, 8:8 + n_out]
    return a, w, n_out, kw


@pytest.mark.gpu
@pytest.mark.parametrize("dt", list(DT))
@pytest.mark.parametrize("name", ["plain", "bias", "rowvec", "ln", "ln_rowvec_res", "silu", "silu_res", "geglu", "geglu_rowvec_res", "res"])
def test_gemm_bit_identical_across_tile_widths(name, dt):
    ops, lib = _ops()
    dtype, M = DT[dt], 1500
    a, w, n_out, kw = _gemm_operands(name, dtype, M)
    outs = {}
    for bn in WIDTHS:
        o = _Out(M, n_out, dtype)
        _at_width(lib, bn, lambda: ops.gemm(a, w, o.view, **kw))
        outs[bn] = o.done(f"gemm {name} bn={bn}")
    for bn in WIDTHS[1:]:
        nd = int((outs[bn] != outs[64]).sum())
        assert nd == 0, f"gemm {name} {dt}: {nd} elements differ between tile widths 64 and {bn}"


@pytest.mark.gpu
@pytest.mark.parametrize("dt", list(DT))
@pytest.mark.parametrize("kind", ["conv3x3", "stride2", "subpixel"])
def test_conv_bit_identical_across_tile_widths(kind, dt):
    ops, lib = _ops()
    dtype, B, H, W, Cin, Cout = DT[dt], 2, 30, 22, 128, 320
    x = _randn((B * H * W, Cin), 210, dtype=dtype)
    w = _randn((Cout, Cin, 3, 3), 211, 1 / math.sqrt(9 * Cin))
    wp = w.to(dtype).permute(0, 2, 3, 1).reshape(Cout, -1).contiguous()
    bias, rv = _randn((Cout,), 212, 0.2), _randn((B, Cout), 213, 0.5)
    if kind == "conv3x3":
        rows, fn = B * H * W, lambda o: ops.conv3x3(x, B, H, W, wp, o, bias=bias, rowvec=rv)
    elif kind == "stride2":
        rows, fn = B * 15 * 11, lambda o: ops.conv3x3_stride2(x, B, H, W, wp, o, 1, bias=bias)
    else:
        wf = ops.fold_upsample_weights(w, dtype)
        rows, fn = B * 4 * H * W, lambda o: ops.upsample2x_conv3x3(x, B, H, W, wf, o, bias=bias)
    outs = {}
    for bn in WIDTHS:
        o = _Out(rows, Cout, dtype)
        _at_width(lib, bn, lambda: fn(o.view))
        outs[bn] = o.done(f"{kind} bn={bn}")
    for bn in WIDTHS[1:]:
        nd = int((outs[bn] != outs[64]).sum())
        assert nd == 0, f"{kind} {dt}: {nd} elements differ between tile widths 64 and {bn}"


def _nan(*ts):
    """NaN-fill the outputs before each kernel pair: a kernel that wrote nothing fails instead of comparing stale bits."""
    for t in ts:
        t.fill_(math.nan)


def _pick_bn(m_tiles, N, num_kb, sms, geglu=False):
    """pick_bn's cost model (supir_b200/csrc/gemm.cu, pick_bn): used here only to choose batch sizes that land on different
    tile widths."""
    if geglu and N >= 256:
        return 128
    best, best_cost = 160, 1e30
    for bn, per_col, overhead in ((256, 1.21, 7620.0), (160, 1.0, 3140.0), (128, 1.34, 5460.0), (64, 1.57, 1120.0)):
        if bn > 64 and N <= bn // 2:
            continue
        rounds = -(-(m_tiles * -(-N // bn)) // sms)
        cost = rounds * (per_col * bn * num_kb + overhead)
        if cost < best_cost - 1e-9:
            best, best_cost = bn, cost
    return best


@pytest.mark.gpu
@pytest.mark.parametrize("dt", list(DT))
def test_gemm_batch_invariance_at_the_heuristic_width(dt):
    """A rank's share of the batch (images [1, 1 + k) of 6) must give the bits of the single-GPU call, though pick_bn may
    choose another width for it. 1000 rows per image is not a multiple of the 128-row tile: the share starts mid-tile, and
    image boundaries (where the per-image vector changes) fall inside tiles."""
    ops, _ = _ops()
    dtype, rpb, K, N = DT[dt], 1000, 640, 1280
    sms = _sms()
    full_bn = _pick_bn(-(-6 * rpb // 128), N, K // 64, sms)
    k = next((k for k in range(1, 6) if _pick_bn(-(-k * rpb // 128), N, K // 64, sms) != full_bn), None)
    assert k is not None, "no sub-batch lands on another tile width"
    a, w = _randn((6 * rpb, K), 220, dtype=dtype), _randn((N, K), 221, 1 / math.sqrt(K), dtype)
    bias, rv = _randn((N,), 222, 0.2), _randn((6, N), 223, 0.5)
    full = _Out(6 * rpb, N, dtype)
    ops.gemm(a, w, full.view, bias=bias, rowvec=rv, rows_per_batch=rpb)
    part = _Out(k * rpb, N, dtype)
    ops.gemm(a[rpb:(1 + k) * rpb], w, part.view, bias=bias, rowvec=rv[1:1 + k], rows_per_batch=rpb)
    nd = int((part.done("gemm part") != full.done("gemm full")[rpb:(1 + k) * rpb]).sum())
    assert nd == 0, f"{dt}: {nd} elements differ between the {k}-image share and the 6-image batch"


@pytest.mark.gpu
@pytest.mark.parametrize("dt", list(DT))
def test_per_image_kernels_batch_invariance(dt):
    """conv3x3 with rowvec, GroupNorm statistics / apply, ZeroSFT, LayerNorm, both attentions, the small convs and
    linear_small_m: images 1..3 alone give the bits they get inside a batch of 5."""
    ops, _ = _ops()
    dtype, B, H, W, C = DT[dt], 5, 24, 20, 320
    HW = H * W
    s0, s1 = 1, 4
    rs = slice(s0 * HW, s1 * HW)
    x = _randn((B * HW, C), 230, dtype=dtype)
    wp = _randn((C, 9 * C), 231, 1 / math.sqrt(9 * C), dtype)
    rv = _randn((B, C), 232, 0.5)
    full, part = torch.empty(B * HW, C, dtype=dtype, device="cuda"), torch.empty((s1 - s0) * HW, C, dtype=dtype, device="cuda")
    _nan(full, part)
    ops.conv3x3(x, B, H, W, wp, full, rowvec=rv)
    ops.conv3x3(x[rs], s1 - s0, H, W, wp, part, rowvec=rv[s0:s1])
    assert torch.equal(full[rs], part), "conv3x3 with rowvec"
    ws_f = torch.zeros(ops.groupnorm_ws_size(B, HW, C), dtype=torch.float64, device="cuda")
    ws_p = torch.zeros(ops.groupnorm_ws_size(s1 - s0, HW, C), dtype=torch.float64, device="cuda")
    ops.groupnorm_stats(x, B, HW, ws_f)
    ops.groupnorm_stats(x[rs], s1 - s0, HW, ws_p)
    assert torch.equal(ws_f[s0 * 64:s1 * 64], ws_p[:(s1 - s0) * 64]), "GroupNorm statistics"
    g, b = _randn((C,), 233) + 1, _randn((C,), 234)
    _nan(full, part)
    ops.groupnorm_apply(x, B, HW, full, g, b, 1e-5, True, sums=ws_f)
    ops.groupnorm_apply(x[rs], s1 - s0, HW, part, g, b, 1e-5, True, sums=ws_p)
    assert torch.equal(full[rs], part), "GroupNorm apply"
    gb = _randn((B * HW, 2 * C), 235, 0.3, dtype)
    skip = _randn((B * HW, C - 160), 236, dtype=dtype)
    cs = torch.tensor([0.6], device="cuda")
    _nan(full, part)
    ops.zerosft_apply(x, skip, 160, gb, full, B, HW, ws_f, g, b, 1e-5, cs)
    ops.zerosft_apply(x[rs], skip[rs], 160, gb[rs], part, s1 - s0, HW, ws_p, g, b, 1e-5, cs)
    assert torch.equal(full[rs], part), "ZeroSFT"
    _nan(full, part)
    ops.layernorm(x, full, g, b)
    ops.layernorm(x[rs], part, g, b)
    assert torch.equal(full[rs], part), "LayerNorm"
    ctx = _randn((B * 77, C), 237, dtype=dtype)
    _nan(full, part)
    ops.attention(x, ctx, ctx, full, B, 5, HW, 77)
    ops.attention(x[rs], ctx[s0 * 77:s1 * 77], ctx[s0 * 77:s1 * 77], part, s1 - s0, 5, HW, 77)
    assert torch.equal(full[rs], part), "attention"
    if dtype == torch.bfloat16:
        _nan(full, part)
        ops.attention_1head(x[:, :128].contiguous(), x[:, 128:256].contiguous(), x[:, 192:320].contiguous(), full[:, :128], B, HW)
        ops.attention_1head(x[rs, :128].contiguous(), x[rs, 128:256].contiguous(), x[rs, 192:320].contiguous(), part[:, :128],
                            s1 - s0, HW)
        assert torch.equal(full[rs, :128], part[:, :128]), "1-head attention"
    img = _randn((B, 4, H, W), 238)
    wc, bc = _randn((C, 4, 3, 3), 239, 0.3), _randn((C,), 240, 0.1)
    _nan(full, part)
    ops.conv3x3_small_cin(img, wc, bc, full, residual=x)
    ops.conv3x3_small_cin(img[s0:s1], wc, bc, part, residual=x[rs])
    assert torch.equal(full[rs], part), "conv3x3_small_cin"
    wo = _randn((4, 3, 3, C), 241, 0.02)
    co_f, co_p = torch.full((B, 4, H, W), math.nan, device="cuda"), torch.full((s1 - s0, 4, H, W), math.nan, device="cuda")
    ops.conv3x3_small_cout(x, B, H, W, wo, bc[:4], co_f)
    ops.conv3x3_small_cout(x[rs], s1 - s0, H, W, wo, bc[:4], co_p)
    assert torch.equal(co_f[s0:s1], co_p), "conv3x3_small_cout"
    e = _randn((B, 1280), 242)
    we = _randn((1280, 1280), 243, 0.03, dtype)
    lf, lp = torch.full((B, 1280), math.nan, device="cuda"), torch.full((s1 - s0, 1280), math.nan, device="cuda")
    ops.linear_small_m(e, we, bc[:1].expand(1280).contiguous(), lf, silu_in=True, silu_out=2, add=e)
    ops.linear_small_m(e[s0:s1], we, bc[:1].expand(1280).contiguous(), lp, silu_in=True, silu_out=2, add=e[s0:s1])
    assert torch.equal(lf[s0:s1], lp), "linear_small_m (B = 5 takes the 16-row kernel, B = 3 the 4-row one)"
