"""Thin PyTorch-tensor front end of the C ABI: pointer/stride extraction, output allocation, argument checks.

PyTorch owns every buffer (weights, activations, RNG); kernels run on torch's current CUDA stream so that calls can be
captured into CUDA graphs. Channels-last activations are 2-D bf16 tensors [B*H*W, C] whose row stride is the leading
dimension handed to the kernels (column slices of wider buffers are fine).

The ops the diffusion networks use also take fp16 operands (their fp16 compute mode): each picks the bf16 entry point or its
`_f16` twin from the dtype of its 16-bit operands, and refuses operands that mix the two before anything is launched.

FP8 linear layers (the networks' float8_e4m3fn mode): gemm_fp8 multiplies e4m3 operands with one fp32 scale per row of each
(quantize_weight at pack time; quantize_rows / layernorm_quant for the activations) into a bf16 result. FP8 convolutions (the
fp8_convs option of that mode): conv3x3_fp8 takes e4m3 activations with one scale per image (groupnorm_apply_quant) and e4m3
weights with one scale per output channel (quantize_weight of the packed [Cout, 9*Cin] matrix). FP8 attention (the
fp8_attention option): attention_quant_fp8 writes e4m3 Q / K / transposed V and their scales from bf16 q, k, v, and
attention_fp8 runs softmax(Q K^T / 8) V on them into a bf16 result.
"""
import ctypes

import torch

from . import _native
import os

from ._native import ConvGeometry, Epilogue

# strided / sub-pixel convolutions through the implicit-GEMM kernel's geometry mode (supir_conv_geom_bf16); "0" restores the
# im2col buffer (stride 2) and the materialised nearest-2x upsample in front of a plain 3x3 convolution
CONV_GEOM = os.environ.get("SUPIR_B200_CONV_GEOM", "1") != "0"

BF16 = torch.bfloat16
F16 = torch.float16
FP8 = torch.float8_e4m3fn
E4M3_MAX = 448.0


def call(name, *args):
    return _native.call(name, *args)


def _entry(name, *ts):
    """`name` (a bf16 entry point) or its fp16 twin, from the dtype of the 16-bit tensors among `ts` (None and fp32 are
    ignored). Mixing bf16 and fp16 operands in one call is an error."""
    dts = {t.dtype for t in ts if t is not None and t.dtype in (BF16, F16)}
    if len(dts) > 1:
        raise TypeError(f"{name}: operands mix bfloat16 and float16")
    return _native.F16_TWINS[name] if dts == {F16} else name


def _ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise _native.SupirNativeError("supir_b200 kernels need CUDA tensors (there is no CPU fallback)")


def _mat(t, dtype=BF16):
    assert t.dim() == 2 and t.stride(1) == 1 and t.dtype == dtype, (t.shape, t.stride(), t.dtype)
    return t


def _mat16(t):
    """A row-major matrix of 16-bit values (bf16 or fp16)."""
    assert t.dim() == 2 and t.stride(1) == 1 and t.dtype in (BF16, F16), (t.shape, t.stride(), t.dtype)
    return t


class Pool:
    """Free-list of scratch tensors keyed by (dtype, numel). Inside CUDA-graph capture the tensors come from the graph's
    private pool and stay valid for the graph's lifetime; reuse keeps the footprint bounded."""

    def __init__(self):
        self.free = {}
        self.all = []

    def get(self, shape, dtype=BF16, device=None):
        n = 1
        for s in shape:
            n *= int(s)
        key = (dtype, n)
        lst = self.free.get(key)
        if lst:
            return lst.pop().view(*shape)
        t = torch.empty(n, dtype=dtype, device=device or "cuda")
        self.all.append(t)
        return t.view(*shape)

    def put(self, *ts):
        for t in ts:
            if t is None:
                continue
            base = t if t._base is None else t._base
            self.free.setdefault((base.dtype, base.numel()), []).append(base.view(-1))

    def free_bytes(self):
        return sum(k[1] * torch.empty((), dtype=k[0]).element_size() * len(v) for k, v in self.free.items())

    def trim(self):
        """Drop the cached free buffers (they go back to torch's caching allocator); tensors still in use stay with their
        holders. For pools OUTSIDE a CUDA graph only (the tiled VAE: a 256-tile pass touches four resolutions whose scratch
        sizes never recur, and keeping all of them cached would not fit 80 GB)."""
        self.free.clear()
        self.all = []


# ------------------------------------------------------------------------------------------------------------------
# tensor-core ops
# ------------------------------------------------------------------------------------------------------------------
def _epilogue(bias, rowvec, rows_per_batch, residual, act, out_f32, ln=None):
    ep = Epilogue()
    ep.ln_stats = None if ln is None else ln[0].data_ptr()
    ep.ln_colsum = None if ln is None else ln[1].data_ptr()
    ep.bias = None if bias is None else bias.data_ptr()
    ep.rowvec = None if rowvec is None else rowvec.data_ptr()
    ep.rows_per_batch = int(rows_per_batch)
    ep.rowvec_ld = 0 if rowvec is None else int(rowvec.stride(0))
    ep.residual = None if residual is None else residual.data_ptr()
    ep.ldr = 0 if residual is None else int(residual.stride(0))
    ep.act = int(act)
    ep.out_f32 = int(out_f32)
    return ep


def gemm(a, w, out, bias=None, rowvec=None, rows_per_batch=0, residual=None, act=0, ln=None):
    """out[M, N'] = epilogue(a[M, K] @ w[N, K]^T); N' = N/2 for act=2 (GEGLU). `out` may be fp32 or bf16.
    `ln=(stats, colsum)` folds a LayerNorm of `a` into the epilogue (see supir_epilogue in include/supir_b200.h): `a` is the
    raw activation, `w` carries gamma, `bias` carries W beta + bias, stats comes from layernorm_stats().
    a / w / residual / a 16-bit out are all bf16 or all fp16."""
    name = _entry("supir_gemm_bf16", a, w, out, residual)
    _need_cuda(a, w, out)
    _mat16(a), _mat16(w)
    M, K = a.shape
    N = w.shape[0]
    assert w.shape[1] == K and out.shape[0] == M and out.shape[1] == (N // 2 if act == 2 else N), (a.shape, w.shape, out.shape)
    if ln is not None:
        assert ln[0].dtype == torch.float32 and ln[0].shape == (M, 2) and ln[0].is_contiguous() and ln[1].shape == (N,)
    ep = _epilogue(bias, rowvec, rows_per_batch, residual, act, out.dtype == torch.float32, ln)
    call(name, _ptr(a), a.stride(0), _ptr(w), w.stride(0), _ptr(out), out.stride(0), M, N, K,
         ctypes.byref(ep), _stream())
    return out


def e4m3_row_scales(x):
    """(scale, inverse) per row of an fp32 matrix, the quantization of every FP8 operand: scale = amax / 448 and
    inverse = 448 / amax (both 1 for an all-zero row); codes = (x * inverse).to(float8_e4m3fn)."""
    amax = x.abs().amax(dim=1)
    pos = amax > 0
    one, fmax = torch.ones_like(amax), torch.full_like(amax, E4M3_MAX)
    # tensor / tensor: IEEE-rounded divisions, as in the kernels (torch divides by a Python scalar as a product with its
    # reciprocal, which rounds twice)
    return torch.where(pos, amax / fmax, one), torch.where(pos, fmax / torch.where(pos, amax, one), one)


def quantize_weight(w):
    """Pack-time FP8 weight: (e4m3 codes [N, K], fp32 scale [N]), one scale per output channel (row) of the bf16 matrix the
    bf16 pack would use."""
    wf = w.detach().to(BF16).to(torch.float32)
    scale, inv = e4m3_row_scales(wf)
    return (wf * inv[:, None]).to(FP8).contiguous(), scale.contiguous()


def gemm_fp8(a_q, a_scale, w_q, w_scale, out, bias=None, residual=None, act=0, ln=None):
    """out[M, N'] = epilogue(a_scale[m] * w_scale[n] * (a_q[M, K] @ w_q[N, K]^T)) (supir_gemm_fp8): e4m3 operands, fp32 row
    scales, bf16 `out` / `residual`; N' = N/2 for act=2 (GEGLU). There is no folded LayerNorm: quantize the normalised rows
    with layernorm_quant instead."""
    if ln is not None:
        raise ValueError("gemm_fp8: no folded LayerNorm (ln=); quantize the normalised activations with layernorm_quant")
    if a_q.dtype != FP8 or w_q.dtype != FP8:
        raise TypeError(f"gemm_fp8: operands must both be float8_e4m3fn (got {a_q.dtype}, {w_q.dtype})")
    if out.dtype != BF16 or (residual is not None and residual.dtype != BF16):
        raise TypeError("gemm_fp8: out and residual are bfloat16")
    if a_scale.dtype != torch.float32 or w_scale.dtype != torch.float32:
        raise TypeError("gemm_fp8: scales are float32")
    _need_cuda(a_q, a_scale, w_q, w_scale, out)
    _mat(a_q, FP8), _mat(w_q, FP8)
    M, K = a_q.shape
    N = w_q.shape[0]
    assert w_q.shape[1] == K and out.shape[0] == M and out.shape[1] == (N // 2 if act == 2 else N), (a_q.shape, w_q.shape, out.shape)
    assert a_scale.shape == (M,) and w_scale.shape == (N,) and a_scale.is_contiguous() and w_scale.is_contiguous()
    ep = _epilogue(bias, None, 0, residual, act, False)
    call("supir_gemm_fp8", _ptr(a_q), a_q.stride(0), _ptr(a_scale), _ptr(w_q), w_q.stride(0), _ptr(w_scale), _ptr(out), out.stride(0),
         M, N, K, ctypes.byref(ep), _stream())
    return out


def quantize_rows(x, q, scale):
    """Row quantization of a bf16 matrix for gemm_fp8: q (e4m3, x's shape) and scale (fp32 [rows]) per e4m3_row_scales."""
    if x.dtype != BF16 or q.dtype != FP8 or scale.dtype != torch.float32:
        raise TypeError(f"quantize_rows: bfloat16 -> float8_e4m3fn + float32 (got {x.dtype}, {q.dtype}, {scale.dtype})")
    _need_cuda(x, q, scale)
    _mat(x), _mat(q, FP8)
    assert q.shape == x.shape and scale.shape == (x.shape[0],) and scale.is_contiguous()
    call("supir_quantize_rows", _ptr(x), x.stride(0), _ptr(q), q.stride(0), _ptr(scale), x.shape[0], x.shape[1], _stream())
    return q, scale


def conv3x3(x, B, H, W, wp, out, bias=None, rowvec=None, residual=None, act=0):
    """3x3/s1/p1 conv on NHWC: x [B*H*W, Cin] (row stride = ld), wp [Cout, 9*Cin] packed (kh, kw, cin)."""
    name = _entry("supir_conv3x3_bf16", x, wp, out, residual)
    _need_cuda(x, wp, out)
    _mat16(x), _mat16(wp)
    Cin = x.shape[1]
    Cout = wp.shape[0]
    assert x.shape[0] == B * H * W and wp.shape[1] == 9 * Cin and wp.is_contiguous() and out.shape == (B * H * W, Cout)
    ep = _epilogue(bias, rowvec, 0, residual, act, out.dtype == torch.float32)
    call(name, _ptr(x), x.stride(0), _ptr(wp), _ptr(out), out.stride(0), B, H, W, Cin, Cout,
         ctypes.byref(ep), _stream())
    return out


def conv3x3_fp8(x_q, x_scale, B, H, W, w_q, w_scale, out, bias=None, rowvec=None, residual=None, act=0):
    """3x3/s1/p1 conv on e4m3 operands (supir_conv3x3_fp8): x_q [B*H*W, Cin] NHWC codes with one fp32 scale per image,
    x_scale [B]; w_q [Cout, 9*Cin] codes packed like conv3x3's weight with one fp32 scale per output channel, w_scale [Cout];
    out[p, n] = epilogue(x_scale[image of p] * w_scale[n] * acc) with conv3x3's bf16 epilogue (bias, rowvec, SiLU, residual)."""
    if x_q.dtype != FP8 or w_q.dtype != FP8:
        raise TypeError(f"conv3x3_fp8: operands must both be float8_e4m3fn (got {x_q.dtype}, {w_q.dtype})")
    if out.dtype != BF16 or (residual is not None and residual.dtype != BF16):
        raise TypeError("conv3x3_fp8: out and residual are bfloat16")
    if x_scale.dtype != torch.float32 or w_scale.dtype != torch.float32:
        raise TypeError("conv3x3_fp8: scales are float32")
    if act not in (0, 1):
        raise ValueError("conv3x3_fp8: act is 0 (none) or 1 (SiLU)")
    _need_cuda(x_q, x_scale, w_q, w_scale, out)
    _mat(x_q, FP8), _mat(w_q, FP8)
    Cin, Cout = x_q.shape[1], w_q.shape[0]
    assert x_q.shape[0] == B * H * W and w_q.shape[1] == 9 * Cin and w_q.is_contiguous() and out.shape == (B * H * W, Cout), \
        (x_q.shape, w_q.shape, out.shape, B, H, W)
    assert x_scale.shape == (B,) and w_scale.shape == (Cout,) and x_scale.is_contiguous() and w_scale.is_contiguous()
    ep = _epilogue(bias, rowvec, 0, residual, act, False)
    call("supir_conv3x3_fp8", _ptr(x_q), x_q.stride(0), _ptr(x_scale), _ptr(w_q), _ptr(w_scale), _ptr(out), out.stride(0), B, H, W,
         Cin, Cout, ctypes.byref(ep), _stream())
    return out


def conv_geom(x, B, Hin, Win, wp, out, geom, bias=None, act=0):
    """General small-kernel convolution (see supir_conv_geometry): x [B*Hin*Win, Cin], wp [Cout, kh*kw*Cin], out [B*out_H*out_W, Cout]."""
    name = _entry("supir_conv_geom_bf16", x, wp, out)
    _need_cuda(x, wp, out)
    _mat16(x), _mat16(wp)
    Cin, Cout = x.shape[1], wp.shape[0]
    g = ConvGeometry(**geom)
    assert x.shape[0] == B * Hin * Win and wp.shape[1] == g.kh * g.kw * Cin and wp.is_contiguous()
    assert out.shape == (B * g.out_H * g.out_W, Cout), (out.shape, B, g.out_H, g.out_W, Cout)
    ep = _epilogue(bias, None, 0, None, act, out.dtype == torch.float32)
    call(name, _ptr(x), x.stride(0), _ptr(wp), _ptr(out), out.stride(0), B, Hin, Win, Cin, Cout, ctypes.byref(g),
         ctypes.byref(ep), _stream())
    return out


def conv3x3_stride2(x, B, H, W, wp, out, pad_lo, bias=None):
    """3x3 stride-2 convolution: pad_lo = 1 is Conv2d(stride=2, padding=1) (openaimodel.py:196-210); pad_lo = 0 is the VAE's
    F.pad(0,1,0,1) + Conv2d(stride=2, padding=0) (model.py:81-85). The TMA gathers every second input pixel: no im2col."""
    Ho, Wo = (H + 2 * pad_lo - 3) // 2 + 1 if pad_lo else (H + 1 - 3) // 2 + 1, (W + 2 * pad_lo - 3) // 2 + 1 if pad_lo else (W + 1 - 3) // 2 + 1
    geom = dict(kh=3, kw=3, stride=2, off_y=-pad_lo, off_x=-pad_lo, Hout=Ho, Wout=Wo, out_sy=1, out_sx=1, out_oy=0, out_ox=0,
                out_H=Ho, out_W=Wo)
    return conv_geom(x, B, H, W, wp, out, geom, bias=bias)


def fold_upsample_weights(w, dtype=BF16):
    """[Cout, Cin, 3, 3] -> four packed [Cout, 2*2*Cin] `dtype` matrices, index py*2+px: a 3x3 convolution of the nearest-2x
    upsampled image equals, for the output pixels of parity (py, px), a 2x2 convolution of the LOW-resolution image whose taps
    are sums of the 3x3 taps that fall on the same source pixel (rows: py=0 -> {0},{1,2}; py=1 -> {0,1},{2}; same for columns)."""
    wf = w.detach().to(dtype).to(torch.float32)            # the values the reference's 16-bit convolution multiplies
    sets = {0: ((0,), (1, 2)), 1: ((0, 1), (2,))}
    out = []
    for py in (0, 1):
        for px in (0, 1):
            taps = []
            for a in (0, 1):
                for b in (0, 1):
                    acc = 0
                    for ky in sets[py][a]:
                        for kx in sets[px][b]:
                            acc = acc + wf[:, :, ky, kx]
                    taps.append(acc)                        # [Cout, Cin]
            out.append(torch.stack(taps, 1).reshape(w.shape[0], -1).to(dtype).contiguous())
    return out


def upsample2x_conv3x3(x, B, H, W, wfold, out, bias=None):
    """conv3x3(nearest_2x(x)) (openaimodel.py:131-151; model.py:64-68) as four sub-pixel 2x2 convolutions on x [B*H*W, Cin]
    writing the interleaved pixels of out [B*2H*2W, Cout]; wfold from fold_upsample_weights."""
    for py in (0, 1):
        for px in (0, 1):
            geom = dict(kh=2, kw=2, stride=1, off_y=py - 1, off_x=px - 1, Hout=H, Wout=W, out_sy=2, out_sx=2, out_oy=py, out_ox=px,
                        out_H=2 * H, out_W=2 * W)
            conv_geom(x, B, H, W, wfold[py * 2 + px], out, geom, bias=bias)
    return out


def attention(q, k, v, out, B, heads, Lq, Lk, scale=None):
    name = _entry("supir_attention_bf16", q, k, v, out)
    _need_cuda(q, k, v, out)
    for t in (q, k, v, out):
        _mat16(t)
    d = q.shape[1] // heads
    call(name, _ptr(q), q.stride(0), _ptr(k), k.stride(0), _ptr(v), v.stride(0), _ptr(out),
         out.stride(0), B, heads, Lq, Lk, d, float(scale if scale is not None else d ** -0.5), _stream())
    return out


def attention_vt_ld(Lk):
    """Row length of attention_quant_fp8's transposed V codes: Lk rounded up to a multiple of 16 bytes."""
    return -(-int(Lk) // 16) * 16


def attention_quant_fp8(q, k, v, B, heads, Lq, Lk, q8, sq, k8, sk, vt8, sv, amax_ws):
    """attention_fp8's operands from bf16 q [B*Lq, >= heads*64] and k, v [B*Lk, ...] (column slices are fine; see
    supir_attention_quant_fp8): q8 (e4m3, q's shape) with sq fp32 [B*Lq, heads] per (token, head); k8 (k's shape) with sk
    [B, heads] per (image, head); vt8 e4m3 [B, heads, 64, attention_vt_ld(Lk)] (V transposed, keys permuted inside every group
    of 32, zero padded) with sv [B, heads, 64] per (image, head, channel). amax_ws: int32 [B * heads * 65] scratch."""
    if q.dtype != BF16 or k.dtype != BF16 or v.dtype != BF16:
        raise TypeError(f"attention_quant_fp8: q, k, v are bfloat16 (got {q.dtype}, {k.dtype}, {v.dtype})")
    if q8.dtype != FP8 or k8.dtype != FP8 or vt8.dtype != FP8:
        raise TypeError("attention_quant_fp8: q8, k8, vt8 are float8_e4m3fn")
    if sq.dtype != torch.float32 or sk.dtype != torch.float32 or sv.dtype != torch.float32 or amax_ws.dtype != torch.int32:
        raise TypeError("attention_quant_fp8: scales are float32, amax_ws int32")
    _need_cuda(q, k, v, q8, sq, k8, sk, vt8, sv, amax_ws)
    for t in (q, k, v):
        _mat(t)
    _mat(q8, FP8), _mat(k8, FP8)
    C = heads * 64
    assert q.shape == (B * Lq, C) and k.shape == (B * Lk, C) and v.shape == (B * Lk, C), (q.shape, k.shape, v.shape)
    assert q8.shape == q.shape and k8.shape == k.shape, (q8.shape, k8.shape)
    ld_vt = _vt_ld(vt8, B, heads, Lk)
    assert sq.shape == (B * Lq, heads) and sk.shape == (B, heads) and sv.shape == (B, heads, 64) and amax_ws.shape == (B * heads * 65,)
    assert sq.is_contiguous() and sk.is_contiguous() and sv.is_contiguous() and amax_ws.is_contiguous()
    call("supir_attention_quant_fp8", _ptr(q), q.stride(0), _ptr(k), k.stride(0), _ptr(v), v.stride(0), _ptr(q8), q8.stride(0),
         _ptr(sq), _ptr(k8), k8.stride(0), _ptr(sk), _ptr(vt8), ld_vt, _ptr(sv), _ptr(amax_ws), B, heads, Lq, Lk, _stream())
    return q8, sq, k8, sk, vt8, sv


def _vt_ld(vt8, B, heads, Lk):
    """Row stride of a [B, heads, 64, >= Lk] transposed-V tensor whose rows are evenly spaced."""
    assert vt8.dim() == 4 and vt8.shape[:3] == (B, heads, 64) and vt8.shape[3] >= Lk and vt8.stride(3) == 1, (vt8.shape, vt8.stride())
    ld = vt8.stride(2)
    assert vt8.stride(1) == 64 * ld and vt8.stride(0) == heads * 64 * ld and ld >= vt8.shape[3], (vt8.shape, vt8.stride())
    return ld


def attention_fp8(q8, sq, k8, sk, vt8, sv, out, B, heads, Lq, Lk, scale=None):
    """out [B*Lq, >= heads*64] bf16 = softmax(Q K^T * scale) V on e4m3 tensor cores from attention_quant_fp8's operands
    (supir_attention_fp8; head_dim 64, scale defaults to 64^-0.5)."""
    if q8.dtype != FP8 or k8.dtype != FP8 or vt8.dtype != FP8:
        raise TypeError(f"attention_fp8: operands are float8_e4m3fn (got {q8.dtype}, {k8.dtype}, {vt8.dtype})")
    if sq.dtype != torch.float32 or sk.dtype != torch.float32 or sv.dtype != torch.float32:
        raise TypeError("attention_fp8: scales are float32")
    if out.dtype != BF16:
        raise TypeError(f"attention_fp8: out is bfloat16 (got {out.dtype})")
    _need_cuda(q8, sq, k8, sk, vt8, sv, out)
    _mat(q8, FP8), _mat(k8, FP8), _mat(out)
    C = heads * 64
    assert q8.shape == (B * Lq, C) and k8.shape == (B * Lk, C) and out.shape == (B * Lq, C), (q8.shape, k8.shape, out.shape)
    ld_vt = _vt_ld(vt8, B, heads, Lk)
    assert sq.shape == (B * Lq, heads) and sk.shape == (B, heads) and sv.shape == (B, heads, 64)
    assert sq.is_contiguous() and sk.is_contiguous() and sv.is_contiguous()
    call("supir_attention_fp8", _ptr(q8), q8.stride(0), _ptr(sq), _ptr(k8), k8.stride(0), _ptr(sk), _ptr(vt8), ld_vt, _ptr(sv),
         _ptr(out), out.stride(0), B, heads, Lq, Lk, 64, float(scale if scale is not None else 0.125), _stream())
    return out


def attention_1head(q, k, v, out, B, L, scale=None):
    """One wide head (head_dim = columns: 512 for the SDXL VAE, 128 / 256 for reduced configs) over L tokens per batch
    element (VAE mid-block attention); q/k/v/out [B*L, head_dim] bf16 (row stride = leading dimension)."""
    _need_cuda(q, k, v, out)
    D = q.shape[1]
    for t in (q, k, v, out):
        _mat(t)
        assert t.shape == (B * L, D), t.shape
    call("supir_attention_1head_bf16", _ptr(q), q.stride(0), _ptr(k), k.stride(0), _ptr(v), v.stride(0), _ptr(out), out.stride(0),
         B, L, D, float(scale if scale is not None else D ** -0.5), _stream())
    return out


# ------------------------------------------------------------------------------------------------------------------
# normalisation
# ------------------------------------------------------------------------------------------------------------------
def groupnorm_ws_size(B, HW, C, groups=32):
    """doubles needed by groupnorm_stats (final sums first, then per-block partials and tickets)."""
    n = int(_native.load().supir_groupnorm_stats_workspace(B, HW, C, groups))
    if n < 0:
        raise _native.SupirNativeError(f"groupnorm: unsupported channel count {C}")
    return n


def groupnorm_stats(x, B, HW, ws, groups=32):
    """ws: float64 workspace of groupnorm_ws_size() elements; ws[:B*groups*2] receives (sum, sumsq) per (image, group)."""
    name = _entry("supir_groupnorm_stats", x)
    _need_cuda(x, ws)
    _mat16(x)
    assert ws.dtype == torch.float64
    call(name, _ptr(x), x.stride(0), B, HW, x.shape[1], groups, _ptr(ws), ws.numel(), _stream())
    return ws


def groupnorm_finalize(sums, n, count, mean, var):
    call("supir_groupnorm_finalize", _ptr(sums), n, float(count), _ptr(mean), _ptr(var), _stream())


def groupnorm_merge_tiles(tile_mean, tile_var, weights, mean, var):
    T, n = tile_mean.shape
    call("supir_groupnorm_merge_tiles", _ptr(tile_mean), _ptr(tile_var), _ptr(weights), T, n, _ptr(mean), _ptr(var), _stream())


def groupnorm_apply(x, B, HW, out, gamma, beta, eps, silu, sums=None, mean=None, var=None, groups=32):
    name = _entry("supir_groupnorm_apply", x, out)
    _need_cuda(x, out)
    _mat16(x), _mat16(out)
    call(name, _ptr(x), x.stride(0), _ptr(out), out.stride(0), B, HW, x.shape[1], groups, _ptr(sums),
         _ptr(mean), _ptr(var), _ptr(gamma), _ptr(beta), float(eps), int(silu), _stream())
    return out


def groupnorm_apply_quant(x, B, HW, q, scale, amax_ws, gamma, beta, eps, silu, sums, groups=32):
    """GroupNorm [+ SiLU] of bf16 x [B*HW, C] written as conv3x3_fp8's operand: q (e4m3, x's shape) and scale (fp32 [B]), one
    scale per image from the amax of the fp32 apply values (no bf16 rounding in between), per e4m3_row_scales of the image's
    values. `sums` from groupnorm_stats; amax_ws: int32 [B] scratch (reset by the call on the stream)."""
    if x.dtype != BF16 or q.dtype != FP8 or scale.dtype != torch.float32 or amax_ws.dtype != torch.int32:
        raise TypeError(f"groupnorm_apply_quant: bfloat16 -> float8_e4m3fn + float32, int32 scratch (got {x.dtype}, {q.dtype}, "
                        f"{scale.dtype}, {amax_ws.dtype})")
    if sums is None or sums.dtype != torch.float64:
        raise TypeError("groupnorm_apply_quant: sums are the float64 output of groupnorm_stats")
    _need_cuda(x, q, scale, amax_ws, sums)
    _mat(x), _mat(q, FP8)
    assert q.shape == x.shape and x.shape[0] == B * HW and scale.shape == (B,) and amax_ws.shape == (B,), (x.shape, q.shape, B, HW)
    assert scale.is_contiguous() and amax_ws.is_contiguous()
    call("supir_groupnorm_apply_quant", _ptr(x), x.stride(0), _ptr(q), q.stride(0), _ptr(scale), _ptr(amax_ws), B, HW, x.shape[1],
         groups, _ptr(sums), _ptr(gamma), _ptr(beta), float(eps), int(silu), _stream())
    return q, scale


def zerosft_apply(h, skip_raw, C1, gamma_beta, out, B, HW, sums, gn_w, gn_b, eps, control_scale, groups=32):
    name = _entry("supir_zerosft_apply", h, skip_raw, gamma_beta, out)
    _need_cuda(h, gamma_beta, out, control_scale)
    call(name, _ptr(h), h.stride(0), _ptr(skip_raw), 0 if skip_raw is None else skip_raw.stride(0), C1,
         _ptr(gamma_beta), gamma_beta.stride(0), _ptr(out), out.stride(0), B, HW, h.shape[1], groups, _ptr(sums),
         _ptr(gn_w), _ptr(gn_b), float(eps), _ptr(control_scale), _stream())
    return out


def layernorm(x, out, gamma, beta, eps=1e-5):
    name = _entry("supir_layernorm_bf16", x, out)
    _need_cuda(x, out)
    _mat16(x), _mat16(out)
    call(name, _ptr(x), x.stride(0), _ptr(out), out.stride(0), x.shape[0], x.shape[1], _ptr(gamma),
         _ptr(beta), float(eps), _stream())
    return out


def layernorm_quant(x, gamma, beta, q, scale, eps=1e-5):
    """LayerNorm of bf16 rows x written as gemm_fp8's operand: q (e4m3, x's shape) and scale (fp32 [rows]) quantized per
    e4m3_row_scales from the fp32 normalised values (no bf16 rounding in between)."""
    if x.dtype != BF16 or q.dtype != FP8 or scale.dtype != torch.float32:
        raise TypeError(f"layernorm_quant: bfloat16 -> float8_e4m3fn + float32 (got {x.dtype}, {q.dtype}, {scale.dtype})")
    _need_cuda(x, q, scale)
    _mat(x), _mat(q, FP8)
    assert q.shape == x.shape and scale.shape == (x.shape[0],) and scale.is_contiguous()
    call("supir_layernorm_quant", _ptr(x), x.stride(0), _ptr(q), q.stride(0), _ptr(scale), x.shape[0], x.shape[1], _ptr(gamma),
         _ptr(beta), float(eps), _stream())
    return q, scale


def layernorm_stats(x, stats, eps=1e-5):
    """stats[r] = (rstd, mean * rstd) of row r of x (fp32 [rows, 2]) for gemm(..., ln=(stats, colsum))."""
    name = _entry("supir_layernorm_stats", x)
    _need_cuda(x, stats)
    _mat16(x)
    assert stats.dtype == torch.float32 and stats.shape == (x.shape[0], 2) and stats.is_contiguous()
    call(name, _ptr(x), x.stride(0), x.shape[0], x.shape[1], float(eps), _ptr(stats), _stream())
    return stats


def fold_layernorm(w, bias, gamma, beta, dtype=BF16):
    """Weights of `Linear(LayerNorm(x))` for the folded form: (`dtype` W * gamma, fp32 colsum of that, fp32 W beta + bias)."""
    wf = w.detach().to(dtype).to(torch.float32)                # the values the reference's 16-bit matmul sees
    wg = (wf * gamma.detach().to(torch.float32)[None, :]).to(dtype).contiguous()
    colsum = wg.to(torch.float32).sum(dim=1).contiguous()
    b2 = wf @ beta.detach().to(torch.float32)
    if bias is not None:
        b2 = b2 + bias.detach().to(dtype).to(torch.float32)
    return wg, colsum, b2.contiguous()


def softmax_rows(S, P, cols, scale):
    _need_cuda(S, P)
    call("supir_softmax_rows", _ptr(S), S.stride(0), _ptr(P), P.stride(0), S.shape[0], cols, float(scale), _stream())
    return P


# ------------------------------------------------------------------------------------------------------------------
# small convs, data movement, embeddings
# ------------------------------------------------------------------------------------------------------------------
def pack_small_cin_weight(w, dtype=BF16):
    """[Cout, Cin, 3, 3] -> `dtype` [Cout, KP] (k = ci*9 + tap, zero padded to a multiple of 64): GEMM operand of the im2col path."""
    cout, taps = w.shape[0], w.shape[1] * 9
    kp = (taps + 63) // 64 * 64
    wp = torch.zeros(cout, kp, dtype=dtype, device=w.device)
    wp[:, :taps] = w.detach().reshape(cout, taps).to(dtype)
    return wp


def conv3x3_small_cin(x_nchw, w, bias, out, residual=None, w_packed=None, pool=None):
    """x_nchw: fp32 [B, Cin, H, W] view with unit stride along W; out NHWC bf16 [B*H*W, Cout].
    With `w_packed` (pack_small_cin_weight) and a scratch `pool`, large images go through im2col + the tensor-core GEMM.
    `out` (and `residual`, `w_packed`) fp16 selects the fp16 kernels: the input is rounded to fp16 instead of bf16."""
    name = _entry("supir_conv3x3_small_cin", out, residual, w_packed)
    _need_cuda(x_nchw, w, out)
    B, Cin, H, W = x_nchw.shape
    assert x_nchw.dtype == torch.float32 and x_nchw.stride(3) == 1 and w.dtype == torch.float32 and w.is_contiguous()
    if w_packed is not None and pool is not None and B * H * W >= 16384 and out.shape[1] >= 64:
        kp = w_packed.shape[1]
        cols = pool.get((B * H * W, kp), w_packed.dtype)
        call(_entry("supir_im2col_3x3_small_cin", cols), _ptr(x_nchw), x_nchw.stride(0), x_nchw.stride(1), x_nchw.stride(2), _ptr(cols),
             cols.stride(0), B, H, W, Cin, kp, _stream())
        gemm(cols, w_packed, out, bias=bias, residual=residual)
        pool.put(cols)
        return out
    call(name, _ptr(x_nchw), x_nchw.stride(0), x_nchw.stride(1), x_nchw.stride(2), _ptr(w), _ptr(bias),
         _ptr(residual), 0 if residual is None else residual.stride(0), _ptr(out), out.stride(0), B, H, W, Cin, out.shape[1],
         _stream())
    return out


def pack_small_cout_weight(w, bias, dtype=BF16):
    """[Cout <= 8, Cin, 3, 3] -> (`dtype` [8, 9*Cin] in conv3x3's (kh, kw, cin) order, fp32 bias[8]), zero rows beyond Cout."""
    cout, cin = w.shape[0], w.shape[1]
    wp = torch.zeros(8, 9 * cin, dtype=dtype, device=w.device)
    wp[:cout] = w.detach().permute(0, 2, 3, 1).reshape(cout, -1).to(dtype)
    b8 = torch.zeros(8, dtype=torch.float32, device=w.device)
    if bias is not None:
        b8[:cout] = bias.detach().to(dtype).to(torch.float32)
    return wp, b8


def conv3x3_small_cout(x, B, H, W, w, bias, out_nchw, crop=None, packed=None, pool=None):
    """x NHWC bf16 [B*H*W, Cin]; out_nchw fp32 [B, Cout, h, w] view (unit stride along w) receiving the crop window.
    With `packed` (pack_small_cout_weight) and a scratch `pool`, large images run on the tensor cores (Cout padded to 8).
    x (and packed[0]) fp16 selects the fp16 kernels."""
    name = _entry("supir_conv3x3_small_cout", x, None if packed is None else packed[0])
    _need_cuda(x, w, out_nchw)
    _mat16(x)
    y0, x0, ch, cw = crop if crop is not None else (0, 0, H, W)
    assert out_nchw.dtype == torch.float32 and out_nchw.stride(3) == 1 and tuple(out_nchw.shape[2:]) == (ch, cw)
    if packed is not None and pool is not None and B * H * W >= 16384 and x.shape[1] % 64 == 0:
        tmp = pool.get((B * H * W, 8), x.dtype)
        conv3x3(x, B, H, W, packed[0], tmp, bias=packed[1])
        call(_entry("supir_nhwc_bf16_crop_to_nchw_f32", tmp), _ptr(tmp), tmp.stride(0), _ptr(out_nchw), out_nchw.stride(0), out_nchw.stride(1),
             out_nchw.stride(2), B, H, W, out_nchw.shape[1], y0, x0, ch, cw, _stream())
        pool.put(tmp)
        return out_nchw
    call(name, _ptr(x), x.stride(0), _ptr(w), _ptr(bias), _ptr(out_nchw), out_nchw.stride(0),
         out_nchw.stride(1), out_nchw.stride(2), B, H, W, x.shape[1], out_nchw.shape[1], y0, x0, ch, cw, _stream())
    return out_nchw


def conv1x1_small_nchw(x, w, bias, out, in_scale=1.0):
    _need_cuda(x, w, out)
    assert x.is_contiguous() and out.is_contiguous() and x.dtype == torch.float32
    B, Cin = x.shape[0], x.shape[1]
    HW = x.numel() // (B * Cin)
    call("supir_conv1x1_small_nchw", _ptr(x), _ptr(w), _ptr(bias), _ptr(out), B, Cin, out.shape[1], HW, float(in_scale), _stream())
    return out


def upsample2x(x, B, H, W, out):
    call("supir_upsample_nearest2x", _ptr(x), x.stride(0), _ptr(out), out.stride(0), B, H, W, x.shape[1], _stream())
    return out


def im2col_s2(x, B, H, W, out, Ho, Wo, pad_lo):
    assert out.is_contiguous() and out.shape == (B * Ho * Wo, 9 * x.shape[1])
    call("supir_im2col_3x3_s2", _ptr(x), x.stride(0), _ptr(out), B, H, W, x.shape[1], Ho, Wo, pad_lo, _stream())
    return out


def copy2d(src, dst):
    call("supir_copy2d_bf16", _ptr(src), src.stride(0), _ptr(dst), dst.stride(0), src.shape[0], src.shape[1], _stream())
    return dst


def axpy(a, y, out, scale):
    call(_entry("supir_axpy_bf16", a, y, out), _ptr(a), a.stride(0), _ptr(y), y.stride(0), _ptr(out), out.stride(0), a.shape[0], a.shape[1],
         _ptr(scale), _stream())
    return out


def nchw_f32_to_nhwc_bf16(x, out):
    B, C = x.shape[0], x.shape[1]
    assert x.is_contiguous() and x.dtype == torch.float32
    call("supir_nchw_f32_to_nhwc_bf16", _ptr(x), _ptr(out), out.stride(0), B, C, x.numel() // (B * C), _stream())
    return out


def nhwc_bf16_to_nchw_f32(x, B, C, HW, out):
    assert out.is_contiguous() and out.dtype == torch.float32
    call("supir_nhwc_bf16_to_nchw_f32", _ptr(x), x.stride(0), _ptr(out), B, C, HW, _stream())
    return out


def f32_to_bf16(x, out):
    assert x.is_contiguous() and out.is_contiguous() and out.dtype == BF16
    call("supir_f32_to_bf16", _ptr(x), _ptr(out), x.numel(), _stream())
    return out


def f32_to_f16(x, out):
    assert x.is_contiguous() and out.is_contiguous() and out.dtype == F16
    call("supir_f32_to_f16", _ptr(x), _ptr(out), x.numel(), _stream())
    return out


def f32_to_16(x, out):
    """out = x rounded to out's dtype: f32_to_bf16 or f32_to_f16."""
    return (f32_to_f16 if out.dtype == F16 else f32_to_bf16)(x, out)


def timestep_embedding(t, out):
    call("supir_timestep_embedding", _ptr(t), _ptr(out), out.shape[0], out.shape[1], _stream())
    return out


def linear_small_m(x, w, bias, out, silu_in=False, silu_out=False, add=None):
    """w bf16 or fp16; the input and the result are rounded to w's dtype where autocast would round them."""
    name = _entry("supir_linear_small_m", w)
    _need_cuda(x, w, out)
    assert x.dtype == torch.float32 and out.dtype == torch.float32 and w.dtype in (BF16, F16) and w.is_contiguous()
    for r0 in range(0, x.shape[0], 16):     # the kernel keeps <= 16 rows in registers; larger batches go in slices
        xs, os_ = x[r0:r0 + 16], out[r0:r0 + 16]
        ad = None if add is None else add[r0:r0 + 16]
        call(name, _ptr(xs), x.stride(0), _ptr(w), _ptr(bias), _ptr(os_), out.stride(0), xs.shape[0], w.shape[0],
             w.shape[1], int(silu_in), int(silu_out), _ptr(ad), 0 if ad is None else add.stride(0), _stream())
    return out


def channel_std_mean(x):
    """(unbiased std, mean) per channel over dims [0, 2, 3] of a contiguous fp32 NCHW tensor — torch.std_mean(x, [0, 2, 3],
    keepdim=True) — from the deterministic fp64 plane sums of supir_plane_stats; the C-element finalisation stays on the device."""
    _need_cuda(x)
    assert x.dtype == torch.float32 and x.is_contiguous() and x.dim() == 4
    N, C = x.shape[:2]
    planes, hw = N * C, x.shape[2] * x.shape[3]
    n = int(_native.load().supir_plane_stats_workspace(planes))
    ws = torch.empty(n, dtype=torch.float64, device=x.device)
    call("supir_plane_stats", _ptr(x), planes, hw, _ptr(ws), n, _stream())
    s = ws[:2 * planes].view(N, C, 2).sum(0)
    cnt = float(N * hw)
    mean = s[:, 0] / cnt
    var = (s[:, 1] - s[:, 0] * s[:, 0] / cnt) / (cnt - 1.0)
    return var.clamp_min(0).sqrt().float().view(1, C, 1, 1), mean.float().view(1, C, 1, 1)


# ------------------------------------------------------------------------------------------------------------------
# text conditioner (textenc.cu)
# ------------------------------------------------------------------------------------------------------------------
def gather_rows_f32(table, idx, out, pos=None, L=0):
    """out[r] = table[idx[r]] (+ pos[r % L]); table / pos / out fp32 matrices, idx int32 [rows]."""
    _need_cuda(table, idx, out, pos)
    assert table.dtype == torch.float32 and out.dtype == torch.float32 and idx.dtype == torch.int32 and idx.is_contiguous()
    assert table.dim() == 2 and out.dim() == 2 and table.stride(1) == 1 and out.stride(1) == 1 and out.shape == (idx.numel(), table.shape[1])
    assert pos is None or (pos.dtype == torch.float32 and pos.stride(1) == 1 and pos.shape[1] == table.shape[1] and pos.shape[0] >= L > 0)
    call("supir_gather_rows_f32", _ptr(table), table.stride(0), table.shape[0], _ptr(idx), _ptr(pos), 0 if pos is None else pos.stride(0),
         int(L), _ptr(out), out.stride(0), out.shape[0], table.shape[1], _stream())
    return out


def layernorm_f32(x, gamma, beta, eps=1e-5, out_bf16=None, out_f32=None):
    """LayerNorm of fp32 rows x [rows, C] into a bf16 and / or an fp32 matrix."""
    _need_cuda(x, out_bf16, out_f32)
    assert x.dtype == torch.float32 and x.dim() == 2 and x.stride(1) == 1 and (out_bf16 is not None or out_f32 is not None)
    assert out_bf16 is None or (_mat(out_bf16).shape == x.shape)
    assert out_f32 is None or (_mat(out_f32, torch.float32).shape == x.shape)
    call("supir_layernorm_f32", _ptr(x), x.stride(0), _ptr(out_bf16), 0 if out_bf16 is None else out_bf16.stride(0), _ptr(out_f32),
         0 if out_f32 is None else out_f32.stride(0), x.shape[0], x.shape[1], _ptr(gamma), _ptr(beta), float(eps), _stream())
    return out_bf16 if out_bf16 is not None else out_f32


def attention_small(q, k, v, out, B, heads, L, causal=True, scale=None):
    """Short-sequence (L <= 128) attention with head_dim 64 and an optional causal mask; q/k/v/out bf16 [B*L, >= heads*64]."""
    _need_cuda(q, k, v, out)
    for t in (q, k, v, out):
        _mat(t)
        assert t.shape[0] == B * L
    d = q.shape[1] // heads
    call("supir_attention_small_bf16", _ptr(q), q.stride(0), _ptr(k), k.stride(0), _ptr(v), v.stride(0), _ptr(out), out.stride(0),
         B, heads, L, d, float(scale if scale is not None else d ** -0.5), int(bool(causal)), _stream())
    return out


def activation(x, out, mode):
    """out = GELU(x) (mode 'gelu', exact erf form) or x * sigmoid(1.702 x) (mode 'quick_gelu'); bf16, x and out may alias."""
    _need_cuda(x, out)
    _mat(x), _mat(out)
    assert x.shape == out.shape
    call("supir_activation_bf16", _ptr(x), x.stride(0), _ptr(out), out.stride(0), x.shape[0], x.shape[1],
         {"gelu": 0, "quick_gelu": 1}[mode], _stream())
    return out


# ------------------------------------------------------------------------------------------------------------------
# sampler
# ------------------------------------------------------------------------------------------------------------------
def edm_pre(x, eps, noise_mul, c_in, x_hat, net_in):
    _need_cuda(x, x_hat, net_in)
    assert x.is_contiguous() and x_hat.is_contiguous() and net_in.is_contiguous() and net_in.numel() == 2 * x.numel()
    call("supir_edm_pre", _ptr(x), _ptr(eps), float(noise_mul), float(c_in), _ptr(x_hat), _ptr(net_in), x.numel(), _stream())


def edm_post(x_hat, net_out, x_center, c_out, cfg_scale, restore_mul, sigma_hat, dt, x_next, denoised=None):
    _need_cuda(x_hat, net_out, x_next)
    assert x_hat.is_contiguous() and net_out.is_contiguous() and x_next.is_contiguous()
    assert x_center is None or x_center.is_contiguous()
    call("supir_edm_post", _ptr(x_hat), _ptr(net_out), _ptr(x_center), float(c_out), float(cfg_scale), float(restore_mul),
         float(sigma_hat), float(dt), _ptr(x_next), _ptr(denoised), x_hat.numel(), _stream())


def axpby_f32(a, alpha, b, beta, out):
    _need_cuda(a, out)
    assert a.is_contiguous() and out.is_contiguous() and a.dtype == torch.float32 and (b is None or b.is_contiguous())
    call("supir_axpby_f32", _ptr(a), float(alpha), _ptr(b), float(beta), _ptr(out), a.numel(), _stream())
    return out


def cfg_combine(x, scale, out):
    _need_cuda(x, scale, out)
    N = out.shape[0]
    assert x.is_contiguous() and out.is_contiguous() and x.shape[0] == 2 * N and scale.dtype == torch.float32
    call("supir_cfg_combine", _ptr(x), _ptr(scale), _ptr(out), N, out.numel() // N, _stream())
    return out


def tile_gather(src, windows, tile, out):
    """out[j, n, c] = src[n, c, window j]; src fp32 [N, C, H, W]; out fp32 [nw, N, C, tile, tile]."""
    _need_cuda(src, windows, out)
    assert src.is_contiguous() and out.is_contiguous() and windows.dtype == torch.int32 and src.dtype == torch.float32
    N, C, H, W = src.shape
    call("supir_tile_gather", _ptr(src), _ptr(windows), windows.shape[0], tile, _ptr(out), N, C, H, W, _stream())
    return out


def tile_blend(tiles, windows, tile, weights, out):
    """tiles fp32 [nw, N, C, tile, tile]; windows int32 [nw, 4]; weights fp64 [tile, tile]; out fp32 [N, C, H, W]."""
    _need_cuda(tiles, windows, weights, out)
    assert tiles.is_contiguous() and out.is_contiguous() and windows.dtype == torch.int32 and weights.dtype == torch.float64
    N, C, H, W = out.shape
    call("supir_tile_blend", _ptr(tiles), _ptr(windows), windows.shape[0], tile, _ptr(weights), _ptr(out), N, C, H, W, _stream())
    return out


def gaussian_latent(moments, eps, scale, z):
    B, C2 = moments.shape[0], moments.shape[1]
    assert moments.is_contiguous() and z.is_contiguous()
    call("supir_gaussian_latent", _ptr(moments), _ptr(eps), float(scale), _ptr(z), B, C2 // 2, moments.numel() // (B * C2), _stream())
    return z
