"""Plain-torch CPU stand-ins for the supir_b200.ops kernels (TEST INFRASTRUCTURE — never imported by the product).

They let the HOST-side code — weight packing (fused QKV / K|V matrices, GEGLU interleave, LayerNorm folding, sub-pixel upsample
folding, embedding / context offsets), the module wiring of GLVControl / LightGLVUNet, the VAE step list and its tiled
executor, the samplers' step logic, unit sharding and exchanges — run without a GPU and be compared with the reference's
golden outputs, also under gloo with several ranks. The arithmetic of the real kernels is pinned by the -m gpu tests; these
stand-ins compute in fp32 and round to the 16-bit type at the points where the kernels round, and
tests/test_gpu_kernel_edges.py holds them to the kernels' error bounds on the kernels' inputs."""
import math

import torch
import torch.nn.functional as F

BF = torch.bfloat16


def _bf(x):
    return x.to(BF).float()


def _nchw(x, B, H, W):
    return x.float().reshape(B, H, W, -1).permute(0, 3, 1, 2)


def _nhwc(y):
    B, C, H, W = y.shape
    return y.permute(0, 2, 3, 1).reshape(B * H * W, C)


def _gelu(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def _finish(acc, out, bias, rowvec_rows, residual, act):
    if bias is not None:
        acc = acc + bias
    if rowvec_rows is not None:
        acc = acc + rowvec_rows
    if act == 2:
        v = acc.view(acc.shape[0], -1, 2, 16)
        acc = (_bf(v[:, :, 0]) * _bf(_gelu(_bf(v[:, :, 1])))).reshape(acc.shape[0], -1)
    elif act == 1:
        acc = F.silu(_bf(acc))
    if residual is not None:
        acc = _bf(acc) + residual.float()
    out.copy_(acc.to(out.dtype))
    return out


# ---- tensor-core ops ----
def gemm(a, w, out, bias=None, rowvec=None, rows_per_batch=0, residual=None, act=0, ln=None):
    acc = a.float() @ w.float().t()
    if ln is not None:
        stats, colsum = ln
        acc = stats[:, 0:1] * acc - stats[:, 1:2] * colsum[None, :]
    rv = None
    if rowvec is not None:
        idx = torch.arange(a.shape[0]) // max(int(rows_per_batch), 1)
        rv = rowvec[idx]
    return _finish(acc, out, bias, rv, residual, act)


def conv3x3(x, B, H, W, wp, out, bias=None, rowvec=None, residual=None, act=0):
    Cin, Cout = x.shape[1], wp.shape[0]
    w = wp.float().view(Cout, 3, 3, Cin).permute(0, 3, 1, 2)
    y = _nhwc(F.conv2d(_nchw(x, B, H, W), w, None, padding=1))
    rv = None if rowvec is None else rowvec.float().repeat_interleave(H * W, dim=0)
    return _finish(y, out, bias, rv, residual, act)


def conv_geom(x, B, Hin, Win, wp, out, geom, bias=None, act=0):
    g = dict(geom)
    Cin, Cout = x.shape[1], wp.shape[0]
    w = wp.float().view(Cout, g["kh"], g["kw"], Cin).permute(0, 3, 1, 2)
    pt, pl = -g["off_y"], -g["off_x"]
    assert pt >= 0 and pl >= 0
    need_h = (g["Hout"] - 1) * g["stride"] + g["kh"] - pt
    need_w = (g["Wout"] - 1) * g["stride"] + g["kw"] - pl
    xin = F.pad(_nchw(x, B, Hin, Win), (pl, max(0, need_w - Win), pt, max(0, need_h - Hin)))
    y = F.conv2d(xin, w, None, stride=g["stride"])[:, :, :g["Hout"], :g["Wout"]]
    if bias is not None:
        y = y + bias.view(1, -1, 1, 1)
    if act == 1:
        y = F.silu(_bf(y))
    o = out.view(B, g["out_H"], g["out_W"], Cout)
    o[:, g["out_oy"]::g["out_sy"], g["out_ox"]::g["out_sx"]][:, :g["Hout"], :g["Wout"]] = y.permute(0, 2, 3, 1).to(out.dtype)
    return out


def attention(q, k, v, out, B, heads, Lq, Lk, scale=None):
    d = q.shape[1] // heads
    sp = lambda t, L: t.float().reshape(B, L, heads, d).transpose(1, 2)  # noqa: E731
    o = F.scaled_dot_product_attention(sp(q, Lq), sp(k, Lk), sp(v, Lk), scale=scale)
    out.copy_(o.transpose(1, 2).reshape(B * Lq, heads * d).to(out.dtype))
    return out


def attention_1head(q, k, v, out, B, L, scale=None):
    return attention(q, k, v, out, B, 1, L, L, scale=scale)


# ---- normalisation ----
def groupnorm_ws_size(B, HW, C, groups=32):
    return B * groups * 2 + 8


def groupnorm_stats(x, B, HW, ws, groups=32):
    v = x.double().reshape(B, HW, groups, -1)
    ws[:B * groups * 2] = torch.stack([v.sum(dim=(1, 3)), (v * v).sum(dim=(1, 3))], -1).reshape(-1)
    return ws


def _mean_var(sums, B, groups, count):
    s = sums[:B * groups * 2].reshape(B * groups, 2)
    mean = s[:, 0] / count
    return mean, s[:, 1] / count - mean * mean


def groupnorm_finalize(sums, n, count, mean, var):
    m, v = _mean_var(sums, n, 1, count)
    mean.copy_(m.float())
    var.copy_(v.float())


def groupnorm_merge_tiles(tile_mean, tile_var, weights, mean, var):
    mean.copy_((weights[:, None] * tile_mean).sum(0))
    var.copy_((weights[:, None] * tile_var).sum(0))


def _gn(x, B, HW, gamma, beta, eps, groups, sums, mean, var):
    C = x.shape[1]
    if sums is not None:
        mean, var = _mean_var(sums, B, groups, HW * (C // groups))
    v = x.float().reshape(B, HW, groups, C // groups)
    m = mean.float().reshape(B, 1, groups, 1)
    r = torch.rsqrt(var.float().reshape(B, 1, groups, 1) + eps)
    return ((v - m) * r).reshape(B * HW, C) * gamma.float()[None] + beta.float()[None]


def groupnorm_apply(x, B, HW, out, gamma, beta, eps, silu, sums=None, mean=None, var=None, groups=32):
    y = _gn(x, B, HW, gamma, beta, eps, groups, sums, mean, var)
    out.copy_((F.silu(y) if silu else y).to(out.dtype))
    return out


def zerosft_apply(h, skip_raw, C1, gamma_beta, out, B, HW, sums, gn_w, gn_b, eps, control_scale, groups=32):
    C = h.shape[1]
    normed = _gn(h, B, HW, gn_w, gn_b, eps, groups, sums, None, None)        # fp32: autocast's group_norm returns fp32
    a = normed * (gamma_beta[:, :C].float() + 1.0).to(out.dtype).float() + gamma_beta[:, C:].float()   # (gamma + 1) is a 16-bit tensor
    h_raw = h.float() if skip_raw is None else torch.cat([h[:, :C1].float(), skip_raw.float()], 1)
    cs = float(control_scale.reshape(-1)[0])
    out.copy_((a * cs + h_raw * (1.0 - cs)).to(out.dtype))
    return out


def layernorm(x, out, gamma, beta, eps=1e-5):
    out.copy_(F.layer_norm(x.float(), (x.shape[1],), gamma.float(), beta.float(), eps).to(out.dtype))
    return out


def layernorm_stats(x, stats, eps=1e-5):
    xf = x.float()
    rstd = torch.rsqrt(xf.var(1, unbiased=False) + eps)
    stats[:, 0] = rstd
    stats[:, 1] = xf.mean(1) * rstd
    return stats


# ---- small convs, data movement, embeddings ----
def conv3x3_small_cin(x_nchw, w, bias, out, residual=None, w_packed=None, pool=None):
    y = _nhwc(F.conv2d(x_nchw.to(out.dtype).float(), w.float(), None if bias is None else bias.float(), padding=1))
    if residual is not None:
        y = y.to(out.dtype).float() + residual.float()
    out.copy_(y.to(out.dtype))
    return out


def conv3x3_small_cout(x, B, H, W, w, bias, out_nchw, crop=None, packed=None, pool=None):
    wt = w.float().permute(0, 3, 1, 2)                 # [Cout, 3, 3, Cin] -> [Cout, Cin, 3, 3]
    # fp64 sum, one rounding to x's 16-bit type: up to 9 * 512 products per output, and only <= 8 output channels
    y = F.conv2d(_nchw(x, B, H, W).double(), wt.double(), None if bias is None else bias.double(), padding=1).to(x.dtype).float()
    y0, x0, ch, cw = crop if crop is not None else (0, 0, H, W)
    out_nchw.copy_(y[:, :out_nchw.shape[1], y0:y0 + ch, x0:x0 + cw])
    return out_nchw


def conv1x1_small_nchw(x, w, bias, out, in_scale=1.0):
    out.copy_(_bf(F.conv2d(_bf(x * in_scale), w.float()[:, :, None, None], None if bias is None else bias.float())))
    return out


def timestep_embedding(t, out):
    dim = out.shape[1]
    half = dim // 2
    freqs = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float32) / half)
    args = t.float()[:, None] * freqs[None]
    out.copy_(torch.cat([torch.cos(args), torch.sin(args)], -1))
    return out


def linear_small_m(x, w, bias, out, silu_in=False, silu_out=False, add=None):
    r = lambda t: t.to(w.dtype).float()  # noqa: E731  (rounding points in w's 16-bit type)
    xv = r(x)
    if silu_in:
        xv = r(F.silu(xv))
    v = xv @ w.float().t()
    v = r(v + (0 if bias is None else bias.float()))
    so = int(silu_out)
    if so & 1:
        v = r(F.silu(v))
    if add is not None:
        v = r(v + add)
    if so & 2:
        v = r(F.silu(v))
    out.copy_(v)
    return out


def upsample2x(x, B, H, W, out):
    v = x.reshape(B, H, 1, W, 1, -1).expand(B, H, 2, W, 2, x.shape[1])
    out.copy_(v.reshape(B * 4 * H * W, -1))
    return out


def im2col_s2(x, B, H, W, out, Ho, Wo, pad_lo):
    C = x.shape[1]
    xp = F.pad(x.reshape(B, H, W, C), (0, 0, pad_lo, 2, pad_lo, 2))
    taps = [xp[:, ky:ky + 2 * Ho:2, kx:kx + 2 * Wo:2] for ky in range(3) for kx in range(3)]
    out.copy_(torch.stack(taps, 3).reshape(B * Ho * Wo, 9 * C))
    return out


def f32_to_bf16(x, out):
    out.copy_(x.to(BF))
    return out


def copy2d(src, dst):
    dst.copy_(src)
    return dst


def axpy(a, y, out, scale):
    out.copy_((a.float() + (y.float() * float(scale.reshape(-1)[0])).to(out.dtype).float()).to(out.dtype))
    return out


def gaussian_latent(moments, eps, scale, z):
    mean, logvar = torch.chunk(moments, 2, dim=1)
    v = mean if eps is None else mean + torch.exp(0.5 * torch.clamp(logvar, -30.0, 20.0)) * eps
    z.copy_(scale * v)
    return z


def channel_std_mean(x):
    return torch.std_mean(x, dim=[0, 2, 3], keepdim=True)


# ---- text conditioner ----
def gather_rows_f32(table, idx, out, pos=None, L=0):
    v = table[idx.long().clamp(0, table.shape[0] - 1)]
    if pos is not None:
        v = v + pos[torch.arange(idx.numel()) % L]
    out.copy_(v)
    return out


def layernorm_f32(x, gamma, beta, eps=1e-5, out_bf16=None, out_f32=None):
    y = F.layer_norm(x.float(), (x.shape[1],), gamma.float(), beta.float(), eps)
    if out_bf16 is not None:
        out_bf16.copy_(y.to(BF))
    if out_f32 is not None:
        out_f32.copy_(y)
    return out_bf16 if out_bf16 is not None else out_f32


def attention_small(q, k, v, out, B, heads, L, causal=True, scale=None):
    d = q.shape[1] // heads
    sp = lambda t: t.float().reshape(B, L, heads, d).transpose(1, 2)  # noqa: E731
    o = F.scaled_dot_product_attention(sp(q), sp(k), sp(v), is_causal=bool(causal), scale=scale)
    out.copy_(o.transpose(1, 2).reshape(B * L, heads * d).to(out.dtype))
    return out


def activation(x, out, mode):
    xf = x.float()
    out.copy_((_gelu(xf) if mode == "gelu" else xf * torch.sigmoid(1.702 * xf)).to(out.dtype))
    return out


# ---- sampler ----
def tile_gather(src, windows, tile, out):
    for j, (hi, he, wi, we) in enumerate(windows.tolist()):
        if hi >= 0:
            out[j] = src[:, :, hi:he, wi:we]
    return out


def tile_blend(tiles, windows, tile, weights, out):
    acc = torch.zeros(out.shape, dtype=torch.float32)
    cnt = torch.zeros(out.shape, dtype=torch.float32)
    w = weights.to(torch.float64)
    for j, (hi, he, wi, we) in enumerate(windows.tolist()):
        if hi < 0:
            continue
        acc[:, :, hi:he, wi:we] += (tiles[j].to(torch.float64) * w).to(torch.float32)
        cnt[:, :, hi:he, wi:we] += w.to(torch.float32)
    out.copy_(acc / cnt)
    return out


def edm_pre(x, eps, noise_mul, c_in, x_hat, net_in):
    v = x if eps is None else x + eps * noise_mul
    x_hat.copy_(v)
    net_in.view(2, -1).copy_((v * c_in).reshape(1, -1).expand(2, -1))


def edm_post(x_hat, net_out, x_center, c_out, cfg_scale, restore_mul, sigma_hat, dt, x_next, denoised=None):
    n = x_hat.numel()
    net = net_out.reshape(2, n)
    xh = x_hat.reshape(-1)
    du, dc = net[0] * c_out + xh, net[1] * c_out + xh
    den = du + cfg_scale * (dc - du)
    if x_center is not None:
        den = den - (den - x_center.reshape(-1)) * restore_mul
    x_next.copy_((xh + (xh - den) / sigma_hat * dt).view(x_next.shape))
    if denoised is not None:
        denoised.copy_(den.view(denoised.shape))


def axpby_f32(a, alpha, b, beta, out):
    out.copy_(a * alpha if b is None else a * alpha + b * beta)
    return out


def cfg_combine(x, scale, out):
    u, c = x.chunk(2)
    out.copy_(u + scale.view(-1, *([1] * (x.dim() - 1))) * (c - u))
    return out


_ALL = ["gemm", "conv3x3", "conv_geom", "attention", "attention_1head", "groupnorm_ws_size", "groupnorm_stats", "groupnorm_finalize",
        "groupnorm_merge_tiles", "groupnorm_apply", "zerosft_apply", "layernorm", "layernorm_stats", "conv3x3_small_cin",
        "conv3x3_small_cout", "conv1x1_small_nchw", "timestep_embedding", "linear_small_m", "upsample2x", "im2col_s2", "f32_to_bf16", "copy2d", "axpy",
        "gaussian_latent", "tile_gather", "tile_blend", "edm_pre", "edm_post", "axpby_f32", "cfg_combine",
        "gather_rows_f32", "layernorm_f32", "attention_small", "activation", "channel_std_mean"]


def install(monkeypatch_or_none=None):
    """Replace the kernels of supir_b200.ops by the stand-ins above (and let its scratch pool allocate on the CPU)."""
    from supir_b200 import ops
    me = globals()
    pool_get = ops.Pool.get

    def cpu_get(self, shape, dtype=BF, device=None):
        return pool_get(self, shape, dtype, device or "cpu")

    def setter(obj, name, val):
        if monkeypatch_or_none is not None:
            monkeypatch_or_none.setattr(obj, name, val)
        else:
            setattr(obj, name, val)
    for k in _ALL:
        setter(ops, k, me[k])
    setter(ops.Pool, "get", cpu_get)
