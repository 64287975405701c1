"""Thin PyTorch-tensor front end of the C ABI: pointer/stride extraction, output allocation, argument checks.

PyTorch owns every buffer (weights, activations, RNG); kernels run on torch's current CUDA stream so that calls can be
captured into CUDA graphs. Channels-last activations are 2-D bf16 tensors [B*H*W, C] whose row stride is the leading
dimension handed to the kernels (column slices of wider buffers are fine).
"""
import ctypes

import torch

from . import _native
import os

from ._native import ConvGeometry, Epilogue, call

# strided / sub-pixel convolutions through the implicit-GEMM kernel's geometry mode (supir_conv_geom_bf16); "0" restores the
# im2col buffer (stride 2) and the materialised nearest-2x upsample in front of a plain 3x3 convolution
CONV_GEOM = os.environ.get("SUPIR_B200_CONV_GEOM", "1") != "0"

BF16 = torch.bfloat16


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
    raw activation, `w` carries gamma, `bias` carries W beta + bias, stats comes from layernorm_stats()."""
    _need_cuda(a, w, out)
    _mat(a), _mat(w)
    M, K = a.shape
    N = w.shape[0]
    assert w.shape[1] == K and out.shape[0] == M and out.shape[1] == (N // 2 if act == 2 else N), (a.shape, w.shape, out.shape)
    if ln is not None:
        assert ln[0].dtype == torch.float32 and ln[0].shape == (M, 2) and ln[0].is_contiguous() and ln[1].shape == (N,)
    ep = _epilogue(bias, rowvec, rows_per_batch, residual, act, out.dtype == torch.float32, ln)
    call("supir_gemm_bf16", _ptr(a), a.stride(0), _ptr(w), w.stride(0), _ptr(out), out.stride(0), M, N, K,
         ctypes.byref(ep), _stream())
    return out


def conv3x3(x, B, H, W, wp, out, bias=None, rowvec=None, residual=None, act=0):
    """3x3/s1/p1 conv on NHWC: x [B*H*W, Cin] (row stride = ld), wp [Cout, 9*Cin] packed (kh, kw, cin)."""
    _need_cuda(x, wp, out)
    _mat(x), _mat(wp)
    Cin = x.shape[1]
    Cout = wp.shape[0]
    assert x.shape[0] == B * H * W and wp.shape[1] == 9 * Cin and wp.is_contiguous() and out.shape == (B * H * W, Cout)
    ep = _epilogue(bias, rowvec, 0, residual, act, out.dtype == torch.float32)
    call("supir_conv3x3_bf16", _ptr(x), x.stride(0), _ptr(wp), _ptr(out), out.stride(0), B, H, W, Cin, Cout,
         ctypes.byref(ep), _stream())
    return out


def conv_geom(x, B, Hin, Win, wp, out, geom, bias=None, act=0):
    """General small-kernel convolution (see supir_conv_geometry): x [B*Hin*Win, Cin], wp [Cout, kh*kw*Cin], out [B*out_H*out_W, Cout]."""
    _need_cuda(x, wp, out)
    _mat(x), _mat(wp)
    Cin, Cout = x.shape[1], wp.shape[0]
    g = ConvGeometry(**geom)
    assert x.shape[0] == B * Hin * Win and wp.shape[1] == g.kh * g.kw * Cin and wp.is_contiguous()
    assert out.shape == (B * g.out_H * g.out_W, Cout), (out.shape, B, g.out_H, g.out_W, Cout)
    ep = _epilogue(bias, None, 0, None, act, out.dtype == torch.float32)
    call("supir_conv_geom_bf16", _ptr(x), x.stride(0), _ptr(wp), _ptr(out), out.stride(0), B, Hin, Win, Cin, Cout, ctypes.byref(g),
         ctypes.byref(ep), _stream())
    return out


def conv3x3_stride2(x, B, H, W, wp, out, pad_lo, bias=None):
    """3x3 stride-2 convolution: pad_lo = 1 is Conv2d(stride=2, padding=1) (openaimodel.py:196-210); pad_lo = 0 is the VAE's
    F.pad(0,1,0,1) + Conv2d(stride=2, padding=0) (model.py:81-85). The TMA gathers every second input pixel: no im2col."""
    Ho, Wo = (H + 2 * pad_lo - 3) // 2 + 1 if pad_lo else (H + 1 - 3) // 2 + 1, (W + 2 * pad_lo - 3) // 2 + 1 if pad_lo else (W + 1 - 3) // 2 + 1
    geom = dict(kh=3, kw=3, stride=2, off_y=-pad_lo, off_x=-pad_lo, Hout=Ho, Wout=Wo, out_sy=1, out_sx=1, out_oy=0, out_ox=0,
                out_H=Ho, out_W=Wo)
    return conv_geom(x, B, H, W, wp, out, geom, bias=bias)


def fold_upsample_weights(w):
    """[Cout, Cin, 3, 3] -> four packed [Cout, 2*2*Cin] bf16 matrices, index py*2+px: a 3x3 convolution of the nearest-2x
    upsampled image equals, for the output pixels of parity (py, px), a 2x2 convolution of the LOW-resolution image whose taps
    are sums of the 3x3 taps that fall on the same source pixel (rows: py=0 -> {0},{1,2}; py=1 -> {0,1},{2}; same for columns)."""
    wf = w.detach().to(BF16).to(torch.float32)             # the values the reference's bf16 convolution multiplies
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
            out.append(torch.stack(taps, 1).reshape(w.shape[0], -1).to(BF16).contiguous())
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
    _need_cuda(q, k, v, out)
    for t in (q, k, v, out):
        _mat(t)
    d = q.shape[1] // heads
    call("supir_attention_bf16", _ptr(q), q.stride(0), _ptr(k), k.stride(0), _ptr(v), v.stride(0), _ptr(out),
         out.stride(0), B, heads, Lq, Lk, d, float(scale if scale is not None else d ** -0.5), _stream())
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
    _need_cuda(x, ws)
    _mat(x)
    assert ws.dtype == torch.float64
    call("supir_groupnorm_stats", _ptr(x), x.stride(0), B, HW, x.shape[1], groups, _ptr(ws), ws.numel(), _stream())
    return ws


def groupnorm_finalize(sums, n, count, mean, var):
    call("supir_groupnorm_finalize", _ptr(sums), n, float(count), _ptr(mean), _ptr(var), _stream())


def groupnorm_merge_tiles(tile_mean, tile_var, weights, mean, var):
    T, n = tile_mean.shape
    call("supir_groupnorm_merge_tiles", _ptr(tile_mean), _ptr(tile_var), _ptr(weights), T, n, _ptr(mean), _ptr(var), _stream())


def groupnorm_apply(x, B, HW, out, gamma, beta, eps, silu, sums=None, mean=None, var=None, groups=32):
    _need_cuda(x, out)
    _mat(x), _mat(out)
    call("supir_groupnorm_apply", _ptr(x), x.stride(0), _ptr(out), out.stride(0), B, HW, x.shape[1], groups, _ptr(sums),
         _ptr(mean), _ptr(var), _ptr(gamma), _ptr(beta), float(eps), int(silu), _stream())
    return out


def zerosft_apply(h, skip_raw, C1, gamma_beta, out, B, HW, sums, gn_w, gn_b, eps, control_scale, groups=32):
    _need_cuda(h, gamma_beta, out, control_scale)
    call("supir_zerosft_apply", _ptr(h), h.stride(0), _ptr(skip_raw), 0 if skip_raw is None else skip_raw.stride(0), C1,
         _ptr(gamma_beta), gamma_beta.stride(0), _ptr(out), out.stride(0), B, HW, h.shape[1], groups, _ptr(sums),
         _ptr(gn_w), _ptr(gn_b), float(eps), _ptr(control_scale), _stream())
    return out


def layernorm(x, out, gamma, beta, eps=1e-5):
    _need_cuda(x, out)
    _mat(x), _mat(out)
    call("supir_layernorm_bf16", _ptr(x), x.stride(0), _ptr(out), out.stride(0), x.shape[0], x.shape[1], _ptr(gamma),
         _ptr(beta), float(eps), _stream())
    return out


def layernorm_stats(x, stats, eps=1e-5):
    """stats[r] = (rstd, mean * rstd) of row r of x (fp32 [rows, 2]) for gemm(..., ln=(stats, colsum))."""
    _need_cuda(x, stats)
    _mat(x)
    assert stats.dtype == torch.float32 and stats.shape == (x.shape[0], 2) and stats.is_contiguous()
    call("supir_layernorm_stats", _ptr(x), x.stride(0), x.shape[0], x.shape[1], float(eps), _ptr(stats), _stream())
    return stats


def fold_layernorm(w, bias, gamma, beta):
    """Weights of `Linear(LayerNorm(x))` for the folded form: (bf16 W * gamma, fp32 colsum of that, fp32 W beta + bias)."""
    wf = w.detach().to(BF16).to(torch.float32)                 # the values the reference's bf16 matmul sees
    wg = (wf * gamma.detach().to(torch.float32)[None, :]).to(BF16).contiguous()
    colsum = wg.to(torch.float32).sum(dim=1).contiguous()
    b2 = wf @ beta.detach().to(torch.float32)
    if bias is not None:
        b2 = b2 + bias.detach().to(BF16).to(torch.float32)
    return wg, colsum, b2.contiguous()


def softmax_rows(S, P, cols, scale):
    _need_cuda(S, P)
    call("supir_softmax_rows", _ptr(S), S.stride(0), _ptr(P), P.stride(0), S.shape[0], cols, float(scale), _stream())
    return P


# ------------------------------------------------------------------------------------------------------------------
# small convs, data movement, embeddings
# ------------------------------------------------------------------------------------------------------------------
def pack_small_cin_weight(w):
    """[Cout, Cin, 3, 3] -> bf16 [Cout, KP] (k = ci*9 + tap, zero padded to a multiple of 64): GEMM operand of the im2col path."""
    cout, taps = w.shape[0], w.shape[1] * 9
    kp = (taps + 63) // 64 * 64
    wp = torch.zeros(cout, kp, dtype=BF16, device=w.device)
    wp[:, :taps] = w.detach().reshape(cout, taps).to(BF16)
    return wp


def conv3x3_small_cin(x_nchw, w, bias, out, residual=None, w_packed=None, pool=None):
    """x_nchw: fp32 [B, Cin, H, W] view with unit stride along W; out NHWC bf16 [B*H*W, Cout].
    With `w_packed` (pack_small_cin_weight) and a scratch `pool`, large images go through im2col + the tensor-core GEMM."""
    _need_cuda(x_nchw, w, out)
    B, Cin, H, W = x_nchw.shape
    assert x_nchw.dtype == torch.float32 and x_nchw.stride(3) == 1 and w.dtype == torch.float32 and w.is_contiguous()
    if w_packed is not None and pool is not None and B * H * W >= 16384 and out.shape[1] >= 64:
        kp = w_packed.shape[1]
        cols = pool.get((B * H * W, kp))
        call("supir_im2col_3x3_small_cin", _ptr(x_nchw), x_nchw.stride(0), x_nchw.stride(1), x_nchw.stride(2), _ptr(cols),
             cols.stride(0), B, H, W, Cin, kp, _stream())
        gemm(cols, w_packed, out, bias=bias, residual=residual)
        pool.put(cols)
        return out
    call("supir_conv3x3_small_cin", _ptr(x_nchw), x_nchw.stride(0), x_nchw.stride(1), x_nchw.stride(2), _ptr(w), _ptr(bias),
         _ptr(residual), 0 if residual is None else residual.stride(0), _ptr(out), out.stride(0), B, H, W, Cin, out.shape[1],
         _stream())
    return out


def pack_small_cout_weight(w, bias):
    """[Cout <= 8, Cin, 3, 3] -> (bf16 [8, 9*Cin] in conv3x3's (kh, kw, cin) order, fp32 bias[8]), zero rows beyond Cout."""
    cout, cin = w.shape[0], w.shape[1]
    wp = torch.zeros(8, 9 * cin, dtype=BF16, device=w.device)
    wp[:cout] = w.detach().permute(0, 2, 3, 1).reshape(cout, -1).to(BF16)
    b8 = torch.zeros(8, dtype=torch.float32, device=w.device)
    if bias is not None:
        b8[:cout] = bias.detach().to(BF16).to(torch.float32)
    return wp, b8


def conv3x3_small_cout(x, B, H, W, w, bias, out_nchw, crop=None, packed=None, pool=None):
    """x NHWC bf16 [B*H*W, Cin]; out_nchw fp32 [B, Cout, h, w] view (unit stride along w) receiving the crop window.
    With `packed` (pack_small_cout_weight) and a scratch `pool`, large images run on the tensor cores (Cout padded to 8)."""
    _need_cuda(x, w, out_nchw)
    _mat(x)
    y0, x0, ch, cw = crop if crop is not None else (0, 0, H, W)
    assert out_nchw.dtype == torch.float32 and out_nchw.stride(3) == 1 and tuple(out_nchw.shape[2:]) == (ch, cw)
    if packed is not None and pool is not None and B * H * W >= 16384 and x.shape[1] % 64 == 0:
        tmp = pool.get((B * H * W, 8))
        conv3x3(x, B, H, W, packed[0], tmp, bias=packed[1])
        call("supir_nhwc_bf16_crop_to_nchw_f32", _ptr(tmp), tmp.stride(0), _ptr(out_nchw), out_nchw.stride(0), out_nchw.stride(1),
             out_nchw.stride(2), B, H, W, out_nchw.shape[1], y0, x0, ch, cw, _stream())
        pool.put(tmp)
        return out_nchw
    call("supir_conv3x3_small_cout", _ptr(x), x.stride(0), _ptr(w), _ptr(bias), _ptr(out_nchw), out_nchw.stride(0),
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
    call("supir_axpy_bf16", _ptr(a), a.stride(0), _ptr(y), y.stride(0), _ptr(out), out.stride(0), a.shape[0], a.shape[1],
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
    assert x.is_contiguous() and out.is_contiguous()
    call("supir_f32_to_bf16", _ptr(x), _ptr(out), x.numel(), _stream())
    return out


def timestep_embedding(t, out):
    call("supir_timestep_embedding", _ptr(t), _ptr(out), out.shape[0], out.shape[1], _stream())
    return out


def linear_small_m(x, w, bias, out, silu_in=False, silu_out=False, add=None):
    _need_cuda(x, w, out)
    assert x.dtype == torch.float32 and out.dtype == torch.float32 and w.dtype == BF16 and w.is_contiguous()
    for r0 in range(0, x.shape[0], 16):     # the kernel keeps <= 16 rows in registers; larger batches go in slices
        xs, os_ = x[r0:r0 + 16], out[r0:r0 + 16]
        ad = None if add is None else add[r0:r0 + 16]
        call("supir_linear_small_m", _ptr(xs), x.stride(0), _ptr(w), _ptr(bias), _ptr(os_), out.stride(0), xs.shape[0], w.shape[0],
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
