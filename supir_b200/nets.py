"""GLVControl / LightGLVUNet for the H100 backend.

Same constructor parameters and state_dict key names as the reference classes (SUPIR/modules/SUPIR_v0.py:155-666,
sgm/modules/diffusionmodules/openaimodel.py:506-961, sgm/modules/attention.py:196-635) so the reference's YAML configs and
checkpoints load unchanged — but the torch modules below only OWN parameters. Nothing here runs a torch op on the hot
path: `pack(dtype)` converts the weights once into the kernel layouts (bf16 or fp16, K-major, fused QKV / KV / GEGLU /
gamma|beta matrices, fp32 biases) and `run()` issues hand-written sm_90a kernels through the C ABI (supir_b200/ops.py) on
channels-last activations of that dtype (torch.autocast(bfloat16) or autocast(float16) numerics). `pack(float8_e4m3fn)` is
the bf16 pack except for the Linear layers inside every BasicTransformerBlock, which hold e4m3 weights with per-row scales and
run on FP8 tensor cores (see `linear`); `pack(float8_e4m3fn, fp8_convs=True)` also runs the two 3x3 convolutions of every
ResBlock on them (see `ResBlock.run`), and `fp8_attention=True` the self-attentions and ZeroCrossAttn (see `attention`).
Options the SUPIR configs never use raise NotImplementedError.
"""
import os

import torch
import torch.nn as nn

from . import ops
from .ops import BF16

# LayerNorm -> Linear pairs (norm1 -> QKV, norm2 -> to_q) run as ONE statistics pass + a GEMM whose epilogue applies the
# normalisation (ops.fold_layernorm); "0" restores the stand-alone LayerNorm kernel in front of those GEMMs.
FUSE_LN = os.environ.get("SUPIR_B200_FUSE_LN", "1") != "0"

GN_EPS_UNET = 1e-5   # GroupNorm32 (sgm/modules/diffusionmodules/util.py:258-276)
GN_EPS_ATTN = 1e-6   # attention.Normalize (sgm/modules/attention.py:122-125)


class Act:
    """Channels-last activation: t is a bf16 or fp16 matrix [B*H*W, C] (row stride = leading dimension)."""
    __slots__ = ("t", "B", "H", "W")

    def __init__(self, t, B, H, W):
        self.t, self.B, self.H, self.W = t, B, H, W

    @property
    def C(self):
        return self.t.shape[1]

    @property
    def HW(self):
        return self.H * self.W

    @property
    def rows(self):
        return self.B * self.H * self.W


class Ctx:
    """Per-call execution context: scratch pool, conditioning tensors, device scalars, compute dtype (bf16 or fp16: the
    dtype the networks were packed in, and of every activation `new` allocates)."""

    def __init__(self, pool, B, dtype=BF16):
        self.pool = pool
        self.B = B
        self.dtype = dtype
        self.emb_all = None        # fp32 [B, sum(Cout of all ResBlocks)]
        self.ctx_kv = None         # [B*Lctx, sum(2*inner)] context K|V projections of every cross-attention (compute dtype)
        self.kv_owned = True       # False: ctx_kv belongs to the caller (projected outside the per-step graph)
        self.Lctx = 0
        self.control_scale = None  # fp32 device scalar

    def new(self, rows, cols, dtype=None):
        return self.pool.get((rows, cols), dtype or self.dtype)

    def free(self, *ts):
        self.pool.put(*[t.t if isinstance(t, Act) else t for t in ts])


def _f32(t):
    return t.detach().to(torch.float32).contiguous()


def _bf(t, dtype=BF16):
    """Weights as the 16-bit GEMM operand (`dtype`: bf16, or fp16 for the fp16 compute mode)."""
    return t.detach().to(dtype).contiguous()


def _bias_values(t, dtype):
    """autocast hands the bias to the 16-bit GEMM; keep those values (rounded to `dtype`, bf16 or fp16), stored as fp32 for
    the epilogue."""
    return None if t is None else t.detach().to(dtype).to(torch.float32).contiguous()


def _bias_bf16_values(t):
    return _bias_values(t, BF16)


def linear(ctx, x, w, out, **kw):
    """out = epilogue(x @ w^T) for a packed weight `w`: a 16-bit matrix (ops.gemm), or the (e4m3 codes, row scales) pair of an
    FP8 layer (ops.gemm_fp8), whose input `x` is either such a pair already (layernorm_quant) or a bf16 matrix quantized here
    (quantize_rows: one extra pass over x)."""
    if not isinstance(w, tuple):
        return ops.gemm(x, w, out, **kw)
    if isinstance(x, tuple):
        return ops.gemm_fp8(*x, *w, out, **kw)
    q, sc = ctx.new(x.shape[0], x.shape[1], ops.FP8), ctx.pool.get((x.shape[0],), torch.float32)
    ops.quantize_rows(x, q, sc)
    ops.gemm_fp8(q, sc, *w, out, **kw)
    ctx.pool.put(q, sc)
    return out


def attention(ctx, fp8, q, k, v, out, B, heads, Lq, Lk):
    """softmax(q k^T / 8) v per head into `out`: the 16-bit kernel (ops.attention), or with `fp8` (the fp8_attention option)
    the operand pass (ops.attention_quant_fp8: e4m3 codes and scales of q, k and transposed v) and the e4m3 kernel
    (ops.attention_fp8)."""
    if not fp8:
        return ops.attention(q, k, v, out, B, heads, Lq, Lk)
    get, f32 = ctx.pool.get, torch.float32
    q8, k8 = ctx.new(B * Lq, heads * 64, ops.FP8), ctx.new(B * Lk, heads * 64, ops.FP8)
    vt8 = get((B, heads, 64, ops.attention_vt_ld(Lk)), ops.FP8)
    sq, sk, sv = get((B * Lq, heads), f32), get((B, heads), f32), get((B, heads, 64), f32)
    amax = get((B * heads * 65,), torch.int32)
    ops.attention_quant_fp8(q, k, v, B, heads, Lq, Lk, q8, sq, k8, sk, vt8, sv, amax)
    ops.attention_fp8(q8, sq, k8, sk, vt8, sv, out, B, heads, Lq, Lk)
    ctx.pool.put(q8, k8, vt8, sq, sk, sv, amax)
    return out


def pack_conv3x3(w, dtype=BF16):
    """[Cout, Cin, 3, 3] -> [Cout, 9*Cin] with k = (kh*3 + kw)*Cin + cin (what supir_conv3x3_bf16 / im2col expect)."""
    return _bf(w.detach().permute(0, 2, 3, 1).reshape(w.shape[0], -1), dtype)


# ----------------------------------------------------------------------------------------------------------------------
# parameter shells + kernels drivers
# ----------------------------------------------------------------------------------------------------------------------
class GroupNorm32(nn.GroupNorm):
    pass


def group_norm(ctx, x: Act, norm: nn.GroupNorm, silu, out=None):
    sums = ctx.pool.get((ops.groupnorm_ws_size(x.B, x.HW, x.C),), torch.float64)
    ops.groupnorm_stats(x.t, x.B, x.HW, sums)
    o = out if out is not None else ctx.new(x.rows, x.C)
    ops.groupnorm_apply(x.t, x.B, x.HW, o, norm._w, norm._b, norm.eps, silu, sums=sums)
    ctx.pool.put(sums)
    return Act(o, x.B, x.H, x.W)


def group_norm_silu_quant(ctx, x: Act, norm: nn.GroupNorm):
    """SiLU(GroupNorm(x)) as conv3x3_fp8's operand: (e4m3 codes [rows, C], fp32 scale [B], one per image)."""
    sums = ctx.pool.get((ops.groupnorm_ws_size(x.B, x.HW, x.C),), torch.float64)
    ops.groupnorm_stats(x.t, x.B, x.HW, sums)
    q, sc, amax = ctx.new(x.rows, x.C, ops.FP8), ctx.pool.get((x.B,), torch.float32), ctx.pool.get((x.B,), torch.int32)
    ops.groupnorm_apply_quant(x.t, x.B, x.HW, q, sc, amax, norm._w, norm._b, norm.eps, True, sums)
    ctx.pool.put(sums, amax)
    return q, sc


def pack_norm(n):
    n._w, n._b = _f32(n.weight), _f32(n.bias)


class TimestepEmbedSequential(nn.Sequential):
    def run(self, ctx, h: Act, release_input=False):
        for layer in self:
            nh = layer.run(ctx, h)
            if release_input:
                ctx.free(h)
            release_input = True
            h = nh
        return h


class ConvIn(nn.Conv2d):
    """4 -> model_channels 3x3 conv fed with fp32 NCHW (input_blocks.0.0, input_hint_block.0)."""

    def pack(self, dtype=BF16):
        self._w, self._b = self.weight.detach().to(dtype).to(torch.float32).contiguous(), _bias_values(self.bias, dtype)
        self._wp = ops.pack_small_cin_weight(self.weight, dtype)

    def run_nchw(self, ctx, x_nchw, residual=None):
        B, _, H, W = x_nchw.shape
        out = ctx.new(B * H * W, self.out_channels)
        ops.conv3x3_small_cin(x_nchw, self._w, self._b, out, residual=None if residual is None else residual.t,
                              w_packed=self._wp, pool=ctx.pool)
        return Act(out, B, H, W)


class ResBlock(nn.Module):
    """openaimodel.py:213-356 (no up/down, no scale-shift norm)."""

    def __init__(self, channels, emb_channels, dropout, out_channels=None, use_conv=False, use_scale_shift_norm=False,
                 dims=2, use_checkpoint=False, up=False, down=False, **kw):
        super().__init__()
        if use_conv or use_scale_shift_norm or up or down or dims != 2 or kw.get("skip_t_emb") or kw.get("exchange_temb_dims"):
            raise NotImplementedError("ResBlock option outside SUPIR's configs")
        self.channels, self.out_channels = channels, out_channels or channels
        self.in_layers = nn.Sequential(GroupNorm32(32, channels), nn.SiLU(), nn.Conv2d(channels, self.out_channels, 3, padding=1))
        self.emb_layers = nn.Sequential(nn.SiLU(), nn.Linear(emb_channels, self.out_channels))
        self.out_layers = nn.Sequential(GroupNorm32(32, self.out_channels), nn.SiLU(), nn.Dropout(p=dropout),
                                        nn.Conv2d(self.out_channels, self.out_channels, 3, padding=1))
        self.skip_connection = nn.Identity() if self.out_channels == channels else nn.Conv2d(channels, self.out_channels, 1)
        self.emb_offset = None

    fp8_convs = False   # set by the network's pack(float8_e4m3fn, fp8_convs=True): e4m3 in_layers.2 / out_layers.3

    def pack(self, dtype=BF16):
        pack_norm(self.in_layers[0]), pack_norm(self.out_layers[0])
        # FP8: (e4m3 codes, one scale per output channel) of the bf16 packed matrix [Cout, 9*Cin]; the bf16 copy is not kept
        conv = (lambda w: ops.quantize_weight(pack_conv3x3(w, dtype))) if self.fp8_convs else (lambda w: pack_conv3x3(w, dtype))
        self._w1, self._b1 = conv(self.in_layers[2].weight), _bias_values(self.in_layers[2].bias, dtype)
        self._w2, self._b2 = conv(self.out_layers[3].weight), _bias_values(self.out_layers[3].bias, dtype)
        if isinstance(self.skip_connection, nn.Conv2d):
            self._ws = _bf(self.skip_connection.weight.reshape(self.out_channels, self.channels), dtype)
            self._bs = _bias_values(self.skip_connection.bias, dtype)

    def _norm_silu(self, ctx, x: Act, norm):
        """The input of a 3x3 convolution: an Act, or packed FP8 the (codes, per-image scales) pair of conv3x3_fp8."""
        return group_norm_silu_quant(ctx, x, norm) if self.fp8_convs else group_norm(ctx, x, norm, silu=True)

    def _conv(self, ctx, n, x: Act, w, out, **kw):
        if self.fp8_convs:
            ops.conv3x3_fp8(*n, x.B, x.H, x.W, *w, out, **kw)
            ctx.free(*n)
        else:
            ops.conv3x3(n.t, x.B, x.H, x.W, w, out, **kw)
            ctx.free(n)

    def run(self, ctx, x: Act):
        n1 = self._norm_silu(ctx, x, self.in_layers[0])
        emb = ctx.emb_all[:, self.emb_offset:self.emb_offset + self.out_channels]
        h = ctx.new(x.rows, self.out_channels)
        self._conv(ctx, n1, x, self._w1, h, bias=self._b1, rowvec=emb)
        hA = Act(h, x.B, x.H, x.W)
        n2 = self._norm_silu(ctx, hA, self.out_layers[0])
        ctx.free(hA)
        if isinstance(self.skip_connection, nn.Conv2d):
            skip = ctx.new(x.rows, self.out_channels)
            ops.gemm(x.t, self._ws, skip, bias=self._bs)
        else:
            skip = x.t
        out = ctx.new(x.rows, self.out_channels)
        self._conv(ctx, n2, x, self._w2, out, bias=self._b2, residual=skip)
        if skip is not x.t:
            ctx.free(skip)
        return Act(out, x.B, x.H, x.W)


class Downsample(nn.Module):
    """openaimodel.py:170-210 with use_conv=True: 3x3 stride 2 pad 1."""

    def __init__(self, channels, use_conv, dims=2, out_channels=None, padding=1, **kw):
        super().__init__()
        if not use_conv or dims != 2 or padding != 1:
            raise NotImplementedError("Downsample option outside SUPIR's configs")
        self.channels, self.out_channels = channels, out_channels or channels
        self.op = nn.Conv2d(channels, self.out_channels, 3, stride=2, padding=1)

    def pack(self, dtype=BF16):
        self._w, self._b = pack_conv3x3(self.op.weight, dtype), _bias_values(self.op.bias, dtype)

    def run(self, ctx, x: Act):
        Ho, Wo = (x.H + 2 - 3) // 2 + 1, (x.W + 2 - 3) // 2 + 1
        out = ctx.new(x.B * Ho * Wo, self.out_channels)
        if ops.CONV_GEOM:
            ops.conv3x3_stride2(x.t, x.B, x.H, x.W, self._w, out, 1, bias=self._b)
        else:
            cols = ctx.new(x.B * Ho * Wo, 9 * x.C)
            ops.im2col_s2(x.t, x.B, x.H, x.W, cols, Ho, Wo, 1)
            ops.gemm(cols, self._w, out, bias=self._b)
            ctx.free(cols)
        return Act(out, x.B, Ho, Wo)


class Upsample(nn.Module):
    """openaimodel.py:108-151 with use_conv=True: nearest 2x then 3x3."""

    def __init__(self, channels, use_conv, dims=2, out_channels=None, padding=1, **kw):
        super().__init__()
        if not use_conv or dims != 2 or padding != 1:
            raise NotImplementedError("Upsample option outside SUPIR's configs")
        self.channels, self.out_channels = channels, out_channels or channels
        self.conv = nn.Conv2d(channels, self.out_channels, 3, padding=1)

    def pack(self, dtype=BF16):
        self._b = _bias_values(self.conv.bias, dtype)
        if ops.CONV_GEOM:
            self._wfold = ops.fold_upsample_weights(self.conv.weight, dtype)
        else:
            self._w = pack_conv3x3(self.conv.weight, dtype)

    def run(self, ctx, x: Act):
        out = ctx.new(4 * x.rows, self.out_channels)
        if ops.CONV_GEOM:      # four sub-pixel 2x2 convolutions on the low-resolution input: no 4x buffer, 2.25x fewer FLOPs
            ops.upsample2x_conv3x3(x.t, x.B, x.H, x.W, self._wfold, out, bias=self._b)
        else:
            up = ctx.new(4 * x.rows, x.C)
            ops.upsample2x(x.t, x.B, x.H, x.W, up)
            ops.conv3x3(up, x.B, 2 * x.H, 2 * x.W, self._w, out, bias=self._b)
            ctx.free(up)
        return Act(out, x.B, 2 * x.H, 2 * x.W)


class CrossAttention(nn.Module):
    """attention.py:196-285 / 288-373 (parameters identical for the SDPA and xformers variants)."""

    def __init__(self, query_dim, context_dim=None, heads=8, dim_head=64, dropout=0.0, **kw):
        super().__init__()
        if dim_head != 64:
            raise NotImplementedError("attention kernels are written for head_dim 64 (SDXL)")
        inner = dim_head * heads
        self.is_self = context_dim is None
        context_dim = context_dim or query_dim
        self.heads, self.inner = heads, inner
        self.to_q = nn.Linear(query_dim, inner, bias=False)
        self.to_k = nn.Linear(context_dim, inner, bias=False)
        self.to_v = nn.Linear(context_dim, inner, bias=False)
        self.to_out = nn.Sequential(nn.Linear(inner, query_dim), nn.Dropout(dropout))
        self.kv_offset = None   # column offset inside Ctx.ctx_kv for text cross-attention

    _ln = None      # (gamma, beta) of the LayerNorm in front of the query projection, set by BasicTransformerBlock.pack
    _fp8 = False    # FP8 query / QKV and output projections, set by BasicTransformerBlock.pack
    fp8_attention = False   # softmax(QK^T)V on e4m3 operands, set by the network's pack(float8_e4m3fn, fp8_attention=True)

    def pack(self, dtype=BF16):
        if self._fp8:
            # e4m3 + per-row scales instead of the bf16 matrices (not kept); the text K|V projection stays bf16
            if self.is_self:
                self._wqkv = ops.quantize_weight(torch.cat([self.to_q.weight, self.to_k.weight, self.to_v.weight], 0))
            else:
                self._wq = ops.quantize_weight(self.to_q.weight)
                self._wkv = _bf(torch.cat([self.to_k.weight, self.to_v.weight], 0), dtype)
            self._c1 = self._bq = None
            self._wo, self._bo = ops.quantize_weight(self.to_out[0].weight), _bias_values(self.to_out[0].bias, dtype)
            return
        if self.is_self:
            wqkv = torch.cat([self.to_q.weight, self.to_k.weight, self.to_v.weight], 0)
            if self._ln is not None:
                self._wqkv, self._c1, self._bq = ops.fold_layernorm(wqkv, None, *self._ln, dtype=dtype)
            else:
                self._wqkv, self._c1, self._bq = _bf(wqkv, dtype), None, None
        else:
            if self._ln is not None:
                self._wq, self._c1, self._bq = ops.fold_layernorm(self.to_q.weight, None, *self._ln, dtype=dtype)
            else:
                self._wq, self._c1, self._bq = _bf(self.to_q.weight, dtype), None, None
            self._wkv = _bf(torch.cat([self.to_k.weight, self.to_v.weight], 0), dtype)
        self._wo, self._bo = _bf(self.to_out[0].weight, dtype), _bias_values(self.to_out[0].bias, dtype)

    def _ln_args(self, stats):
        """gemm() keywords of the query-side projection: folded LayerNorm when this module was packed with one."""
        if self._c1 is None:
            assert stats is None, "this CrossAttention was packed without a folded LayerNorm: pass normalised activations"
            return {}
        assert stats is not None, "this CrossAttention folds its LayerNorm: pass the raw activations and their row statistics"
        return dict(bias=self._bq, ln=(stats, self._c1))

    def run_self(self, ctx, xn, x_res, B, L, stats=None):
        """x_res + to_out(attn(xn)); xn, x_res: [B*L, C]. With a folded LayerNorm xn is the RAW input and `stats` its row
        statistics (ops.layernorm_stats); packed FP8, xn is the (codes, scales) pair of the normalised input (see `linear`)."""
        C = self.inner
        qkv = ctx.new(B * L, 3 * C)
        linear(ctx, xn, self._wqkv, qkv, **self._ln_args(stats))
        a = ctx.new(B * L, C)
        attention(ctx, self.fp8_attention, qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], a, B, self.heads, L, L)
        ctx.free(qkv)
        out = ctx.new(B * L, x_res.shape[1])
        linear(ctx, a, self._wo, out, bias=self._bo, residual=x_res)
        ctx.free(a)
        return out

    def run_cross(self, ctx, xn, x_res, B, L, k, v, Lk, residual=True, stats=None):
        C = self.inner
        q = ctx.new(B * L, C)
        linear(ctx, xn, self._wq, q, **self._ln_args(stats))
        a = ctx.new(B * L, C)
        attention(ctx, self.fp8_attention, q, k, v, a, B, self.heads, L, Lk)
        ctx.free(q)
        out = ctx.new(B * L, self.to_out[0].out_features)
        linear(ctx, a, self._wo, out, bias=self._bo, residual=x_res if residual else None)
        ctx.free(a)
        return out


class GEGLU(nn.Module):
    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out * 2)


class FeedForward(nn.Module):
    """attention.py:84-110 with glu=True."""

    def __init__(self, dim, mult=4, dropout=0.0):
        super().__init__()
        inner = int(dim * mult)
        self.inner = inner
        self.net = nn.Sequential(GEGLU(dim, inner), nn.Dropout(dropout), nn.Linear(inner, dim))

    _fp8 = False    # e4m3 GEGLU and output projections, set by BasicTransformerBlock.pack

    def pack(self, dtype=BF16):
        w, b = self.net[0].proj.weight.detach(), self.net[0].proj.bias.detach()
        inner = self.inner
        assert inner % 16 == 0
        # interleave value / gate rows in groups of 16 so that each 32-column accumulator chunk holds both halves (FP8: each
        # row keeps its own scale, so the scales follow the same permutation)
        idx = torch.arange(inner, device=w.device).view(-1, 16)
        perm = torch.cat([idx, idx + inner], dim=1).reshape(-1)
        weight = ops.quantize_weight if self._fp8 else (lambda t: _bf(t, dtype))
        self._w1, self._b1 = weight(w[perm]), _bias_values(b[perm], dtype)
        self._w2, self._b2 = weight(self.net[2].weight), _bias_values(self.net[2].bias, dtype)

    def run(self, ctx, xn, x_res):
        g = ctx.new(x_res.shape[0], self.inner)
        linear(ctx, xn, self._w1, g, bias=self._b1, act=2)
        out = ctx.new(x_res.shape[0], x_res.shape[1])
        linear(ctx, g, self._w2, out, bias=self._b2, residual=x_res)
        ctx.free(g)
        return out


class BasicTransformerBlock(nn.Module):
    """attention.py:376-486."""

    def __init__(self, dim, n_heads, d_head, dropout=0.0, context_dim=None, gated_ff=True, disable_self_attn=False, **kw):
        super().__init__()
        if disable_self_attn or not gated_ff:
            raise NotImplementedError("BasicTransformerBlock option outside SUPIR's configs")
        self.attn1 = CrossAttention(query_dim=dim, heads=n_heads, dim_head=d_head, dropout=dropout)
        self.ff = FeedForward(dim, dropout=dropout)
        self.attn2 = CrossAttention(query_dim=dim, context_dim=context_dim, heads=n_heads, dim_head=d_head, dropout=dropout)
        self.norm1, self.norm2, self.norm3 = nn.LayerNorm(dim), nn.LayerNorm(dim), nn.LayerNorm(dim)

    fp8 = False     # set by the network's pack(float8_e4m3fn): the Linear layers below run on e4m3 operands

    def pack(self, dtype=BF16):
        for n in (self.norm1, self.norm2, self.norm3):
            pack_norm(n)
        # norm1 -> QKV and norm2 -> to_q are folded into those GEMMs (runs before the children's pack(): modules() yields
        # parents first). norm3 stays a kernel: its consumer is the GEGLU GEMM, whose epilogue is already the bound.
        # FP8 folds nothing: the fold would quantize the raw, uncentred rows, whose mean then cancels against mean * colsum
        # after quantization; each LayerNorm writes its normalised rows as e4m3 instead (layernorm_quant).
        self.attn1._fp8 = self.attn2._fp8 = self.ff._fp8 = self.fp8
        self.fuse_ln = FUSE_LN and not self.fp8
        self.attn1._ln = (self.norm1.weight, self.norm1.bias) if self.fuse_ln else None
        self.attn2._ln = (self.norm2.weight, self.norm2.bias) if self.fuse_ln else None

    def run(self, ctx, x, B, L):
        C = self.attn2.inner
        off = self.attn2.kv_offset
        k, v = ctx.ctx_kv[:, off:off + C], ctx.ctx_kv[:, off + C:off + 2 * C]
        if self.fp8:
            nq = (ctx.new(x.shape[0], x.shape[1], ops.FP8), ctx.pool.get((x.shape[0],), torch.float32))
            ops.layernorm_quant(x, self.norm1._w, self.norm1._b, *nq, self.norm1.eps)
            x1 = self.attn1.run_self(ctx, nq, x, B, L)
            ctx.free(x)
            ops.layernorm_quant(x1, self.norm2._w, self.norm2._b, *nq, self.norm2.eps)
            x2 = self.attn2.run_cross(ctx, nq, x1, B, L, k, v, ctx.Lctx)
            ctx.free(x1)
            ops.layernorm_quant(x2, self.norm3._w, self.norm3._b, *nq, self.norm3.eps)
            x3 = self.ff.run(ctx, nq, x2)
            ctx.free(x2, *nq)
            return x3
        n = ctx.new(*x.shape)
        if self.fuse_ln:
            st = ctx.pool.get((x.shape[0], 2), torch.float32)
            ops.layernorm_stats(x, st, self.norm1.eps)
            x1 = self.attn1.run_self(ctx, x, x, B, L, stats=st)
            ctx.free(x)
            ops.layernorm_stats(x1, st, self.norm2.eps)
            x2 = self.attn2.run_cross(ctx, x1, x1, B, L, k, v, ctx.Lctx, stats=st)
            ctx.pool.put(st)
        else:
            ops.layernorm(x, n, self.norm1._w, self.norm1._b)
            x1 = self.attn1.run_self(ctx, n, x, B, L)
            ctx.free(x)
            ops.layernorm(x1, n, self.norm2._w, self.norm2._b)
            x2 = self.attn2.run_cross(ctx, n, x1, B, L, k, v, ctx.Lctx)
        ctx.free(x1)
        ops.layernorm(x2, n, self.norm3._w, self.norm3._b)
        x3 = self.ff.run(ctx, n, x2)
        ctx.free(x2, n)
        return x3


class SpatialTransformer(nn.Module):
    """attention.py:533-635 with use_linear=True."""

    def __init__(self, in_channels, n_heads, d_head, depth=1, dropout=0.0, context_dim=None, disable_self_attn=False,
                 use_linear=False, **kw):
        super().__init__()
        if not use_linear or disable_self_attn:
            raise NotImplementedError("SpatialTransformer option outside SUPIR's configs")
        if isinstance(context_dim, (list, tuple)):
            context_dim = context_dim[0]
        inner = n_heads * d_head
        self.norm = nn.GroupNorm(32, in_channels, eps=GN_EPS_ATTN, affine=True)
        self.proj_in = nn.Linear(in_channels, inner)
        self.transformer_blocks = nn.ModuleList(
            [BasicTransformerBlock(inner, n_heads, d_head, dropout=dropout, context_dim=context_dim) for _ in range(depth)])
        self.proj_out = nn.Linear(inner, in_channels)

    def pack(self, dtype=BF16):
        pack_norm(self.norm)
        self._wi, self._bi = _bf(self.proj_in.weight, dtype), _bias_values(self.proj_in.bias, dtype)
        self._wo, self._bo = _bf(self.proj_out.weight, dtype), _bias_values(self.proj_out.bias, dtype)

    def run(self, ctx, x: Act):
        n = group_norm(ctx, x, self.norm, silu=False)
        t = ctx.new(x.rows, self._wi.shape[0])
        ops.gemm(n.t, self._wi, t, bias=self._bi)
        ctx.free(n)
        for blk in self.transformer_blocks:
            t = blk.run(ctx, t, x.B, x.HW)
        out = ctx.new(x.rows, x.C)
        ops.gemm(t, self._wo, out, bias=self._bo, residual=x.t)
        ctx.free(t)
        return Act(out, x.B, x.H, x.W)


class ZeroSFT(nn.Module):
    """SUPIR_v0.py:62-113."""

    def __init__(self, label_nc, norm_nc, concat_channels=0, norm=True, mask=False):
        super().__init__()
        if not norm or mask:
            raise NotImplementedError("ZeroSFT option outside SUPIR's configs")
        C = norm_nc + concat_channels
        self.label_nc, self.norm_nc, self.concat_channels = label_nc, norm_nc, concat_channels
        self.param_free_norm = GroupNorm32(32, C)
        self.mlp_shared = nn.Sequential(nn.Conv2d(label_nc, 128, 3, padding=1), nn.SiLU())
        self.zero_mul = nn.Conv2d(128, C, 3, padding=1)
        self.zero_add = nn.Conv2d(128, C, 3, padding=1)
        self.zero_conv = nn.Conv2d(label_nc, norm_nc, 1, 1, 0)
        self.pre_concat = concat_channels != 0
        self.mask = mask

    def pack(self, dtype=BF16):
        pack_norm(self.param_free_norm)
        self._ws, self._bs = pack_conv3x3(self.mlp_shared[0].weight, dtype), _bias_values(self.mlp_shared[0].bias, dtype)
        self._wgb = torch.cat([pack_conv3x3(self.zero_mul.weight, dtype), pack_conv3x3(self.zero_add.weight, dtype)], 0).contiguous()
        self._bgb = torch.cat([_bias_values(self.zero_mul.bias, dtype), _bias_values(self.zero_add.bias, dtype)],
                              0).contiguous()
        self._wz = _bf(self.zero_conv.weight.reshape(self.norm_nc, self.label_nc), dtype)
        self._bz = _bias_values(self.zero_conv.bias, dtype)

    def run(self, ctx, c: Act, h: Act, h_ori: Act = None):
        if h_ori is not None and not self.pre_concat:
            raise NotImplementedError("ZeroSFT(h_ori) without concat channels is not used by SUPIR")
        C1 = h_ori.C if h_ori is not None else 0
        C = C1 + h.C
        hcat = ctx.new(h.rows, C)
        if h_ori is not None:
            ops.copy2d(h_ori.t, hcat[:, :C1])
        ops.gemm(c.t, self._wz, hcat[:, C1:], bias=self._bz, residual=h.t)       # h + zero_conv(c)
        actv = ctx.new(h.rows, 128)
        ops.conv3x3(c.t, c.B, c.H, c.W, self._ws, actv, bias=self._bs, act=1)     # SiLU(conv(c))
        gb = ctx.new(h.rows, 2 * C)
        ops.conv3x3(actv, c.B, c.H, c.W, self._wgb, gb, bias=self._bgb)           # gamma | beta
        ctx.free(actv)
        sums = ctx.pool.get((ops.groupnorm_ws_size(h.B, h.HW, C),), torch.float64)
        ops.groupnorm_stats(hcat, h.B, h.HW, sums)
        out = ctx.new(h.rows, C)
        n = self.param_free_norm
        ops.zerosft_apply(hcat, h.t, C1, gb, out, h.B, h.HW, sums, n._w, n._b, n.eps, ctx.control_scale)
        ctx.pool.put(sums)
        ctx.free(hcat, gb)
        return Act(out, h.B, h.H, h.W)


class ZeroCrossAttn(nn.Module):
    """SUPIR_v0.py:116-152."""

    def __init__(self, context_dim, query_dim, zero_out=True, mask=False):
        super().__init__()
        self.attn = CrossAttention(query_dim=query_dim, context_dim=context_dim, heads=query_dim // 64, dim_head=64)
        self.norm1 = GroupNorm32(32, query_dim)
        self.norm2 = GroupNorm32(32, context_dim)
        self.mask = mask

    def pack(self, dtype=BF16):
        pack_norm(self.norm1), pack_norm(self.norm2)

    def run(self, ctx, context: Act, x: Act):
        xn = group_norm(ctx, x, self.norm1, silu=False)
        cn = group_norm(ctx, context, self.norm2, silu=False)
        C = self.attn.inner
        kv = ctx.new(context.rows, 2 * C)
        ops.gemm(cn.t, self.attn._wkv, kv)
        ctx.free(cn)
        o = self.attn.run_cross(ctx, xn.t, None, x.B, x.HW, kv[:, :C], kv[:, C:], context.HW, residual=False)
        ctx.free(xn, kv)
        out = ctx.new(x.rows, x.C)
        ops.axpy(x.t, o, out, ctx.control_scale)
        ctx.free(o)
        return Act(out, x.B, x.H, x.W)


# ----------------------------------------------------------------------------------------------------------------------
# networks
# ----------------------------------------------------------------------------------------------------------------------
def _as_list(v, n):
    return list(v) if isinstance(v, (list, tuple)) or type(v).__name__ == "ListConfig" else n * [v]


class _UNetBase(nn.Module):
    """Shared constructor logic of UNetModel / GLVControl (openaimodel.py:536-961, SUPIR_v0.py:156-483)."""

    def _build_common(self, in_channels, model_channels, num_res_blocks, attention_resolutions, dropout, channel_mult,
                      num_head_channels, transformer_depth, context_dim, adm_in_channels, num_classes, kw):
        unsupported = dict(conv_resample=True, dims=2, use_scale_shift_norm=False, resblock_updown=False,
                           use_new_attention_order=False, n_embed=None, disable_self_attentions=None,
                           num_attention_blocks=None, disable_middle_self_attn=False)
        for k, v in unsupported.items():
            if kw.get(k, v) != v:
                raise NotImplementedError(f"{k}={kw[k]} is outside SUPIR's configs")
        if not kw.get("use_spatial_transformer", False) or not kw.get("use_linear_in_transformer", False):
            raise NotImplementedError("only use_spatial_transformer=True, use_linear_in_transformer=True is supported")
        if kw.get("legacy", True) or num_head_channels == -1:
            raise NotImplementedError("only legacy=False with num_head_channels set is supported")
        if num_classes != "sequential" or adm_in_channels is None:
            raise NotImplementedError("only num_classes='sequential' is supported")
        self.in_channels, self.model_channels = in_channels, model_channels
        self.num_classes = num_classes
        channel_mult = list(channel_mult)
        self.num_res_blocks = _as_list(num_res_blocks, len(channel_mult))
        transformer_depth = _as_list(transformer_depth, len(channel_mult))
        depth_mid = kw.get("transformer_depth_middle") or transformer_depth[-1]
        ted = model_channels * 4
        self.time_embed = nn.Sequential(nn.Linear(model_channels, ted), nn.SiLU(), nn.Linear(ted, ted))
        self.label_emb = nn.Sequential(nn.Sequential(nn.Linear(adm_in_channels, ted), nn.SiLU(), nn.Linear(ted, ted)))

        def st(ch, depth):
            return SpatialTransformer(ch, ch // num_head_channels, num_head_channels, depth=depth, context_dim=context_dim,
                                      use_linear=True)

        self.input_blocks = nn.ModuleList([TimestepEmbedSequential(ConvIn(in_channels, model_channels, 3, padding=1))])
        chans = [model_channels]
        ch, ds = model_channels, 1
        for level, mult in enumerate(channel_mult):
            for _ in range(self.num_res_blocks[level]):
                layers = [ResBlock(ch, ted, dropout, out_channels=mult * model_channels)]
                ch = mult * model_channels
                if ds in attention_resolutions:
                    layers.append(st(ch, transformer_depth[level]))
                self.input_blocks.append(TimestepEmbedSequential(*layers))
                chans.append(ch)
            if level != len(channel_mult) - 1:
                self.input_blocks.append(TimestepEmbedSequential(Downsample(ch, True, out_channels=ch)))
                chans.append(ch)
                ds *= 2
        self.middle_block = TimestepEmbedSequential(ResBlock(ch, ted, dropout), st(ch, depth_mid), ResBlock(ch, ted, dropout))
        return chans, ch, ds, ted, transformer_depth, st

    # ---- packing -----------------------------------------------------------------------------------------------------
    def pack(self, dtype=BF16, fp8_convs=False, fp8_attention=False):
        """Convert parameters into kernel layouts (call again after load_state_dict / .to()). `dtype` is the compute dtype:
        torch.bfloat16, or torch.float16 for the fp16 mode (every 16-bit weight, bias value and activation in fp16), or
        torch.float8_e4m3fn for the FP8 mode: bf16 everywhere except the Linear layers of every BasicTransformerBlock (QKV,
        to_out, the cross-attention's to_q, GEGLU, ff.net.2), which hold e4m3 weights with one fp32 scale per output channel
        and take e4m3 activations with one scale per row. `fp8_convs` (FP8 mode only) also runs the two 3x3 convolutions of
        every ResBlock (in_layers.2, out_layers.3) on e4m3 weights with one scale per output channel and e4m3 activations with
        one scale per image (the GroupNorm + SiLU in front of them writes them). `fp8_attention` (FP8 mode only) runs the
        self-attention of every BasicTransformerBlock and the attention of every ZeroCrossAttn on e4m3 operands (`attention`);
        the text cross-attention (attn2) stays bf16."""
        if dtype not in (BF16, ops.F16, ops.FP8):
            raise ValueError(f"compute dtype {dtype} is not supported (bfloat16, float16 or float8_e4m3fn)")
        if fp8_convs and dtype != ops.FP8:
            raise ValueError(f"fp8_convs needs the float8_e4m3fn compute dtype (got {dtype})")
        if fp8_attention and dtype != ops.FP8:
            raise ValueError(f"fp8_attention needs the float8_e4m3fn compute dtype (got {dtype})")
        fp8 = dtype == ops.FP8
        dtype = BF16 if fp8 else dtype
        res, xattn = [], []
        for m in self.modules():
            if isinstance(m, ResBlock):
                res.append(m)
                m.fp8_convs = bool(fp8_convs)
            if isinstance(m, BasicTransformerBlock):
                xattn.append(m.attn2)
                m.fp8 = fp8
                m.attn1.fp8_attention = bool(fp8_attention)
            if isinstance(m, ZeroCrossAttn):
                m.attn.fp8_attention = bool(fp8_attention)
        off = 0
        for r in res:
            r.emb_offset = off
            off += r.out_channels
        self._emb_w = _bf(torch.cat([r.emb_layers[1].weight for r in res], 0), dtype)
        self._emb_b = torch.cat([_bias_values(r.emb_layers[1].bias, dtype) for r in res], 0).contiguous()
        off = 0
        for a in xattn:
            a.kv_offset = off
            off += 2 * a.inner
        self._ctx_kv_cols = off
        for m in self.modules():
            if m is not self and hasattr(m, "pack") and not isinstance(m, _UNetBase):
                m.pack(dtype)
        # text K|V projection of every cross-attention as ONE weight matrix [sum(2*inner), context_dim]
        self._ctx_w = torch.cat([a._wkv for a in xattn], 0).contiguous()
        te, le = self.time_embed, self.label_emb[0]
        self._te = (_bf(te[0].weight, dtype), _bias_values(te[0].bias, dtype), _bf(te[2].weight, dtype),
                    _bias_values(te[2].bias, dtype))
        self._le = (_bf(le[0].weight, dtype), _bias_values(le[0].bias, dtype), _bf(le[2].weight, dtype),
                    _bias_values(le[2].bias, dtype))
        self._packed_device = self._emb_w.device
        self._packed_dtype = dtype
        self._fp8_linears = fp8
        self._fp8_convs = bool(fp8_convs)
        self._fp8_attention = bool(fp8_attention)
        return self

    def project_context(self, context_16, out):
        """Text K|V of EVERY cross-attention of this network as one GEMM: out[B*Lctx, sum 2*inner] (attention.py:248-251).
        The context and `out` are in the packed compute dtype.
        The context is constant over the sampler steps, so ControlWrapper runs this outside the per-step CUDA graph and
        only when the context changes."""
        return ops.gemm(context_16, self._ctx_w, out)

    def _prepare_ctx(self, ctx, t_f32, context_16, B, Lctx, y_f32, ctx_kv=None):
        """K8: timestep + label embedding MLPs and every ResBlock's emb projection; text K|V for all cross-attentions
        (`ctx_kv`: already projected by project_context)."""
        p = ctx.pool
        temb = p.get((B, self.model_channels), torch.float32)
        ops.timestep_embedding(t_f32, temb)
        ted = self._te[0].shape[0]
        h1, e_t, h2, emb = (p.get((B, ted), torch.float32) for _ in range(4))
        ops.linear_small_m(temb, self._te[0], self._te[1], h1, silu_out=True)
        ops.linear_small_m(h1, self._te[2], self._te[3], e_t)
        ops.linear_small_m(y_f32, self._le[0], self._le[1], h2, silu_out=True)
        # emb = time_embed(t) + label_emb(y) is only consumed through the ResBlocks' SiLU -> Linear: store SiLU(emb) once
        ops.linear_small_m(h2, self._le[2], self._le[3], emb, add=e_t, silu_out=2)
        ctx.emb_all = p.get((B, self._emb_w.shape[0]), torch.float32)
        if B > 16:      # every ResBlock's emb projection at once: [B, 1280] x [sum Cout, 1280]^T — a tensor-core GEMM beyond a few rows
            emb_bf = p.get((B, emb.shape[1]), ctx.dtype)
            ops.f32_to_16(emb, emb_bf)
            ops.gemm(emb_bf, self._emb_w, ctx.emb_all, bias=self._emb_b)
            p.put(emb_bf)
        else:
            ops.linear_small_m(emb, self._emb_w, self._emb_b, ctx.emb_all)
        p.put(temb, h1, e_t, h2, emb)
        ctx.kv_owned = ctx_kv is None
        if ctx_kv is None:
            ctx_kv = self.project_context(context_16, p.get((B * Lctx, self._ctx_kv_cols), ctx.dtype))
        ctx.ctx_kv = ctx_kv
        ctx.Lctx = Lctx

    def _release_ctx(self, ctx):
        ctx.pool.put(ctx.emb_all, ctx.ctx_kv if ctx.kv_owned else None)
        ctx.emb_all = ctx.ctx_kv = None


class GLVControl(_UNetBase):
    """SUPIR/modules/SUPIR_v0.py:155-540: SDXL encoder half + zero hint conv; returns 10 feature maps."""

    def __init__(self, in_channels, model_channels, out_channels, num_res_blocks, attention_resolutions, dropout=0,
                 channel_mult=(1, 2, 4, 8), num_classes=None, num_head_channels=-1, transformer_depth=1, context_dim=None,
                 adm_in_channels=None, input_upscale=1, **kw):
        super().__init__()
        if input_upscale != 1:
            raise NotImplementedError("input_upscale != 1 is outside SUPIR's configs")
        self._build_common(in_channels, model_channels, num_res_blocks, attention_resolutions, dropout, channel_mult,
                           num_head_channels, transformer_depth, context_dim, adm_in_channels, num_classes, kw)
        self.input_hint_block = TimestepEmbedSequential(ConvIn(in_channels, model_channels, 3, padding=1))

    def run(self, ctx, control_x, t_f32, xt, context_16, Lctx, y_f32, ctx_kv=None):
        """control_x, xt: fp32 NCHW. Returns list[Act] (the reference's `hs`)."""
        B = xt.shape[0]
        self._prepare_ctx(ctx, t_f32, context_16, B, Lctx, y_f32, ctx_kv)
        hint = self.input_hint_block[0].run_nchw(ctx, control_x)
        h = self.input_blocks[0][0].run_nchw(ctx, xt, residual=hint)   # conv_in(xt) + guided_hint
        ctx.free(hint)
        hs = [h]
        for blk in list(self.input_blocks)[1:]:
            h = blk.run(ctx, h)
            hs.append(h)
        h = self.middle_block.run(ctx, h)
        hs.append(h)
        self._release_ctx(ctx)
        return hs


class LightGLVUNet(_UNetBase):
    """SUPIR/modules/SUPIR_v0.py:543-666 on top of UNetModel (openaimodel.py:506-1013)."""

    def __init__(self, mode="", project_type="ZeroSFT", project_channel_scale=1, in_channels=4, model_channels=320,
                 out_channels=4, num_res_blocks=2, attention_resolutions=(), dropout=0, channel_mult=(1, 2, 4, 8),
                 num_classes=None, num_head_channels=-1, transformer_depth=1, context_dim=None, adm_in_channels=None, **kw):
        super().__init__()
        chans, ch, ds, ted, transformer_depth, st = self._build_common(
            in_channels, model_channels, num_res_blocks, attention_resolutions, dropout, channel_mult, num_head_channels,
            transformer_depth, context_dim, adm_in_channels, num_classes, kw)
        channel_mult = list(channel_mult)
        self.output_blocks = nn.ModuleList([])
        for level, mult in list(enumerate(channel_mult))[::-1]:
            for i in range(self.num_res_blocks[level] + 1):
                ich = chans.pop()
                layers = [ResBlock(ch + ich, ted, dropout, out_channels=model_channels * mult)]
                ch = model_channels * mult
                if ds in attention_resolutions:
                    layers.append(st(ch, transformer_depth[level]))
                if level and i == self.num_res_blocks[level]:
                    layers.append(Upsample(ch, True, out_channels=ch))
                    ds //= 2
                self.output_blocks.append(TimestepEmbedSequential(*layers))
        self.out = nn.Sequential(GroupNorm32(32, ch), nn.SiLU(), nn.Conv2d(model_channels, out_channels, 3, padding=1))
        self.out_channels = out_channels
        if mode != "XL-base" or project_type != "ZeroSFT":
            raise NotImplementedError("only mode='XL-base', project_type='ZeroSFT' (SUPIR v0) is supported")
        cond_output_channels = [320] * 4 + [640] * 3 + [1280] * 3
        project_channels = [int(c * project_channel_scale) for c in [160] * 4 + [320] * 3 + [640] * 3]
        concat_channels = [320] * 2 + [640] * 3 + [1280] * 4 + [0]
        self.project_modules = nn.ModuleList(
            [ZeroSFT(project_channels[i], cond_output_channels[i], concat_channels=concat_channels[i])
             for i in range(len(cond_output_channels))])
        for i in [6, 3]:
            self.project_modules.insert(i, ZeroCrossAttn(cond_output_channels[i], concat_channels[i]))

    def pack(self, dtype=BF16, fp8_convs=False, fp8_attention=False):
        super().pack(dtype, fp8_convs, fp8_attention)
        dtype = self._packed_dtype
        pack_norm(self.out[0])
        w = self.out[2].weight.detach()
        self._wout = w.to(dtype).to(torch.float32).permute(0, 2, 3, 1).contiguous()     # [Cout, 3, 3, Cin]
        self._bout = _bias_values(self.out[2].bias, dtype)
        self._out_packed = ops.pack_small_cout_weight(w, self.out[2].bias, dtype)
        return self

    def run(self, ctx, x, t_f32, context_16, Lctx, y_f32, control, out_nchw, ctx_kv=None):
        """x fp32 NCHW; control: list[Act] from GLVControl.run; out_nchw: fp32 [B, out_channels, H, W]."""
        B = x.shape[0]
        self._prepare_ctx(ctx, t_f32, context_16, B, Lctx, y_f32, ctx_kv)
        h = self.input_blocks[0][0].run_nchw(ctx, x)
        hs = [h]
        for blk in list(self.input_blocks)[1:]:
            h = blk.run(ctx, h)
            hs.append(h)
        proj = self.project_modules
        adapter, cidx = len(proj) - 1, len(control) - 1
        h = self.middle_block.run(ctx, h)
        nh = proj[adapter].run(ctx, control[cidx], h)
        ctx.free(h, control[cidx])
        h = nh
        adapter -= 1
        cidx -= 1
        for blk in self.output_blocks:
            skip = hs.pop()
            nh = proj[adapter].run(ctx, control[cidx], skip, h)
            ctx.free(h, skip)
            h = nh
            adapter -= 1
            if len(blk) == 3:
                for layer in list(blk)[:2]:
                    nh = layer.run(ctx, h)
                    ctx.free(h)
                    h = nh
                nh = proj[adapter].run(ctx, control[cidx], h)
                ctx.free(h)
                h = nh
                adapter -= 1
                nh = blk[2].run(ctx, h)
                ctx.free(h)
                h = nh
            else:
                h = blk.run(ctx, h, release_input=True)
            ctx.free(control[cidx])
            cidx -= 1
        n = group_norm(ctx, h, self.out[0], silu=True)
        ctx.free(h)
        ops.conv3x3_small_cout(n.t, n.B, n.H, n.W, self._wout, self._bout, out_nchw, packed=self._out_packed, pool=ctx.pool)
        ctx.free(n)
        self._release_ctx(ctx)
        return out_nchw
