"""GPU parity of the individual kernels (through the C ABI) against plain PyTorch fp32 maths / the oracle."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

BF = torch.bfloat16


def _ops():
    from supir_b200 import ops
    return ops


def rnd(shape, seed, scale=1.0):
    return (torch.randn(shape, generator=torch.Generator().manual_seed(seed)) * scale)


def nhwc(x):  # [B,C,H,W] fp32 -> bf16 [B*H*W, C] cuda
    B, C, H, W = x.shape
    return x.permute(0, 2, 3, 1).reshape(B * H * W, C).to(BF).cuda().contiguous()


def from_nhwc(t, B, H, W):
    return t.float().cpu().reshape(B, H, W, -1).permute(0, 3, 1, 2)


def close(got, ref, atol, rtol=2e-2):
    err = (got - ref).abs()
    tol = atol + rtol * ref.abs()
    assert bool((err <= tol).all()), f"max err {err.max().item():.4g} (ref max {ref.abs().max().item():.4g})"


@pytest.mark.parametrize("C,H,W,eps,silu", [(320, 16, 24, 1e-5, True), (1920, 8, 8, 1e-5, True), (640, 12, 12, 1e-6, False),
                                            (128, 30, 20, 1e-6, True), (2560, 4, 4, 1e-5, True)])
def test_groupnorm(C, H, W, eps, silu):
    ops = _ops()
    B = 2
    x = (rnd((B, C, H, W), 1) * 2 + 0.5).to(BF).float()
    g, b = rnd((C,), 2) * 0.2 + 1, rnd((C,), 3) * 0.2
    ref = F.group_norm(x, 32, g, b, eps)
    if silu:
        ref = F.silu(ref)
    xt = nhwc(x)
    sums = torch.zeros(ops.groupnorm_ws_size(B, H * W, C), dtype=torch.float64, device="cuda")
    out = torch.empty_like(xt)
    ops.groupnorm_stats(xt, B, H * W, sums)
    first = sums[:B * 64].clone()
    ops.groupnorm_stats(xt, B, H * W, sums)
    assert torch.equal(first, sums[:B * 64]), "GroupNorm statistics must be bit-reproducible"
    ops.groupnorm_apply(xt, B, H * W, out, g.cuda(), b.cuda(), eps, silu, sums=sums)
    close(from_nhwc(out, B, H, W), ref, 2e-2)
    # explicit mean/var path (tiled VAE)
    mean = torch.empty(B * 32, device="cuda")
    var = torch.empty(B * 32, device="cuda")
    ops.groupnorm_finalize(sums, B * 32, H * W * (C // 32), mean, var)
    r = x.view(B, 32, -1)
    close(mean.cpu(), r.mean(-1).reshape(-1), 1e-4, 1e-4)
    close(var.cpu(), r.var(-1, unbiased=False).reshape(-1), 1e-3, 1e-3)
    out2 = torch.empty_like(xt)
    ops.groupnorm_apply(xt, B, H * W, out2, g.cuda(), b.cuda(), eps, silu, mean=mean, var=var)
    close(from_nhwc(out2, B, H, W), ref, 2e-2)


@pytest.mark.parametrize("C", [640, 1280, 320])
def test_layernorm(C):
    ops = _ops()
    x = (rnd((300, C), 4) * 1.5 + 0.3).to(BF)
    g, b = rnd((C,), 5) * 0.2 + 1, rnd((C,), 6) * 0.2
    ref = F.layer_norm(x.float(), (C,), g, b, 1e-5)
    out = torch.empty(300, C, dtype=BF, device="cuda")
    ops.layernorm(x.cuda(), out, g.cuda(), b.cuda())
    close(out.float().cpu(), ref, 2e-2)


def test_softmax_rows():
    ops = _ops()
    S = rnd((70, 1000), 7) * 4
    P = torch.empty(70, 1008, dtype=BF, device="cuda")
    ops.softmax_rows(S.cuda(), P, 1000, 0.25)
    close(P[:, :1000].float().cpu(), torch.softmax(S * 0.25, -1), 1e-3)


def test_small_convs_and_conv1x1():
    ops = _ops()
    B, H, W = 2, 20, 28
    x = rnd((B, 4, H, W), 8)
    w = (rnd((320, 4, 3, 3), 9) * 0.2).to(BF).float()
    b = (rnd((320,), 10) * 0.1).to(BF).float()
    res = rnd((B, 320, H, W), 11).to(BF)
    ref = F.conv2d(x.to(BF).float(), w, b, padding=1).to(BF).float() + res.float()
    out = torch.empty(B * H * W, 320, dtype=BF, device="cuda")
    ops.conv3x3_small_cin(x.cuda(), w.cuda(), b.cuda(), out, residual=nhwc(res.float()))
    close(from_nhwc(out, B, H, W), ref, 3e-2)
    # strided view (a tile of a larger image)
    big = rnd((B, 3, 40, 50), 12).cuda()
    tile = big[:, :, 5:25, 7:35]
    w3 = (rnd((128, 3, 3, 3), 13) * 0.2).to(BF).float()
    out = torch.empty(B * 20 * 28, 128, dtype=BF, device="cuda")
    ops.conv3x3_small_cin(tile, w3.cuda(), None, out)
    ref = F.conv2d(tile.cpu().to(BF).float(), w3, None, padding=1)
    close(from_nhwc(out, B, 20, 28), ref, 3e-2)
    # Cout small, with crop window
    xin = rnd((B, 128, H, W), 14).to(BF)
    for cout in (3, 4, 8):
        wc = (rnd((cout, 128, 3, 3), 15 + cout) * 0.05).to(BF).float()
        bc = (rnd((cout,), 16) * 0.1).to(BF).float()
        ref = F.conv2d(xin.float(), wc, bc, padding=1).to(BF).float()
        canvas = torch.zeros(B, cout, 30, 40, device="cuda")
        dst = canvas[:, :, 4:4 + 12, 6:6 + 20]
        ops.conv3x3_small_cout(nhwc(xin.float()), B, H, W, wc.permute(0, 2, 3, 1).contiguous().cuda(), bc.cuda(), dst, crop=(3, 5, 12, 20))
        close(dst.cpu(), ref[:, :, 3:15, 5:25], 3e-2)
        assert float(canvas[:, :, :4].abs().max()) == 0.0
    x8 = rnd((B, 8, 9, 11), 20)
    w8, b8 = rnd((8, 8), 21) * 0.3, rnd((8,), 22) * 0.1
    y = torch.empty(B, 8, 9, 11, device="cuda")
    ops.conv1x1_small_nchw(x8.cuda(), w8.cuda(), b8.cuda(), y, in_scale=0.5)
    ref = F.conv2d((x8 * 0.5).to(BF).float(), w8[:, :, None, None], b8)
    close(y.cpu(), ref, 2e-2)


def test_entry_exit_convs_on_tensor_cores_match_cuda_core_kernels():
    """Large images route the Cin<=8 / Cout<=8 convs through im2col + wgmma GEMM / the padded implicit-GEMM conv
    (ops.conv3x3_small_cin / _small_cout with packed weights): same values as the CUDA-core kernels and as torch."""
    ops = _ops()
    pool = ops.Pool()
    B, H, W = 1, 128, 136                           # >= 16384 pixels switches the path on
    big = rnd((B, 4, H + 9, W + 11), 31).cuda()
    tile = big[:, :, 4:4 + H, 6:6 + W]              # strided NCHW view, like a VAE tile
    w = (rnd((320, 4, 3, 3), 32) * 0.2).to(BF).float()
    b = (rnd((320,), 33) * 0.1).to(BF).float()
    res = rnd((B * H * W, 320), 34).to(BF).cuda()
    o_cc = torch.empty(B * H * W, 320, dtype=BF, device="cuda")
    o_tc = torch.empty_like(o_cc)
    ops.conv3x3_small_cin(tile, w.cuda(), b.cuda(), o_cc, residual=res)
    ops.conv3x3_small_cin(tile, w.cuda(), b.cuda(), o_tc, residual=res, w_packed=ops.pack_small_cin_weight(w.cuda()), pool=pool)
    ref = F.conv2d(tile.cpu().to(BF).float(), w, b, padding=1).to(BF).float() + from_nhwc(res, B, H, W).float()
    close(from_nhwc(o_tc, B, H, W), ref, 3e-2)
    close(o_tc.float().cpu(), o_cc.float().cpu(), 2e-2)
    xin = rnd((B, 128, H, W), 35).to(BF)
    for cout in (3, 4, 8):
        wc = (rnd((cout, 128, 3, 3), 36 + cout) * 0.05).to(BF).float()
        bc = (rnd((cout,), 37) * 0.1).to(BF).float()
        ref = F.conv2d(xin.float(), wc, bc, padding=1).to(BF).float()
        canvas = torch.zeros(B, cout, H + 10, W + 10, device="cuda")
        dst = canvas[:, :, 5:5 + 100, 7:7 + 90]
        ops.conv3x3_small_cout(nhwc(xin.float()), B, H, W, wc.permute(0, 2, 3, 1).contiguous().cuda(), bc.cuda(), dst,
                               crop=(9, 11, 100, 90), packed=ops.pack_small_cout_weight(wc.cuda(), bc.cuda()), pool=pool)
        close(dst.cpu(), ref[:, :, 9:109, 11:101], 3e-2)
        assert float(canvas[:, :, :5].abs().max()) == 0.0 and float(canvas[:, :, :, :7].abs().max()) == 0.0


def test_upsample_im2col_copy_axpy_layout():
    ops = _ops()
    B, C, H, W = 2, 64, 6, 10
    x = rnd((B, C, H, W), 23).to(BF)
    xt = nhwc(x.float())
    up = torch.empty(B * 4 * H * W, C, dtype=BF, device="cuda")
    ops.upsample2x(xt, B, H, W, up)
    assert torch.equal(from_nhwc(up, B, 2 * H, 2 * W), F.interpolate(x.float(), scale_factor=2, mode="nearest"))
    for pad_lo, (Ho, Wo) in [(1, ((H - 1) // 2 + 1, (W - 1) // 2 + 1)), (0, ((H + 1 - 3) // 2 + 1, (W + 1 - 3) // 2 + 1))]:
        cols = torch.empty(B * Ho * Wo, 9 * C, dtype=BF, device="cuda")
        ops.im2col_s2(xt, B, H, W, cols, Ho, Wo, pad_lo)
        xp = F.pad(x.float(), (1, 1, 1, 1)) if pad_lo == 1 else F.pad(x.float(), (0, 1, 0, 1))
        ref = F.unfold(xp, 3, stride=2).view(B, C, 9, Ho * Wo).permute(0, 3, 2, 1).reshape(B * Ho * Wo, 9 * C)
        assert torch.equal(cols.float().cpu(), ref)
    dst = torch.zeros(B * H * W, 2 * C, dtype=BF, device="cuda")
    ops.copy2d(xt, dst[:, C:])
    assert torch.equal(dst[:, C:], xt) and float(dst[:, :C].abs().max()) == 0
    y = nhwc(rnd((B, C, H, W), 24))
    s = torch.tensor([0.7], device="cuda")
    out = torch.empty_like(xt)
    ops.axpy(xt, y, out, s)
    close(out.float().cpu(), xt.float().cpu() + (y.float().cpu() * 0.7).to(BF).float(), 2e-2)
    back = torch.empty(B, C, H, W, device="cuda")
    ops.nhwc_bf16_to_nchw_f32(xt, B, C, H * W, back)
    assert torch.equal(back.cpu(), x.float())
    fwd = torch.empty(B * H * W, C, dtype=BF, device="cuda")
    ops.nchw_f32_to_nhwc_bf16(x.float().cuda(), fwd)
    assert torch.equal(fwd, xt)


def test_embedding_and_small_linear():
    from oracle.unet import timestep_embedding
    ops = _ops()
    t = torch.tensor([999.0, 401.0, 0.0, 13.0])
    out = torch.empty(4, 320, device="cuda")
    ops.timestep_embedding(t.cuda(), out)
    close(out.cpu(), timestep_embedding(t, 320), 2e-3, 0)
    x = rnd((4, 2816), 25)
    w = (rnd((1280, 2816), 26) * 0.02).to(BF)
    b = (rnd((1280,), 27) * 0.1).to(BF).float()
    add = rnd((4, 1280), 28).to(BF).float()
    y = torch.empty(4, 1280, device="cuda")
    ops.linear_small_m(x.cuda(), w.cuda(), b.cuda(), y, silu_in=True, silu_out=True, add=add.cuda())
    ref = F.silu(F.linear(F.silu(x.to(BF).float()).to(BF).float(), w.float(), b).to(BF).float()).to(BF).float() + add
    close(y.cpu(), ref, 3e-2)


def test_zerosft_apply_matches_oracle_formula():
    ops = _ops()
    B, H, W, C1, C2 = 2, 8, 12, 64, 64
    C = C1 + C2
    h = rnd((B, C, H, W), 30).to(BF).float()
    skip_raw = rnd((B, C2, H, W), 31).to(BF).float()
    gamma, beta = rnd((B, C, H, W), 32).to(BF).float() * 0.3, rnd((B, C, H, W), 33).to(BF).float() * 0.3
    gw, gb = rnd((C,), 34) * 0.2 + 1, rnd((C,), 35) * 0.2
    cs = 0.7
    h_raw = torch.cat([h[:, :C1], skip_raw], 1)
    ref = (F.group_norm(h, 32, gw, gb, 1e-5) * (gamma + 1) + beta) * cs + h_raw * (1 - cs)
    ht = nhwc(h)
    sums = torch.zeros(ops.groupnorm_ws_size(B, H * W, C), dtype=torch.float64, device="cuda")
    ops.groupnorm_stats(ht, B, H * W, sums)
    gbt = torch.cat([nhwc(gamma), nhwc(beta)], 1).contiguous()
    out = torch.empty_like(ht)
    ops.zerosft_apply(ht, nhwc(skip_raw), C1, gbt, out, B, H * W, sums, gw.cuda(), gb.cuda(), 1e-5, torch.tensor([cs], device="cuda"))
    close(from_nhwc(out, B, H, W), ref, 3e-2)


def test_sampler_kernels():
    from oracle import sampler as osamp
    ops = _ops()
    n = (2, 4, 10, 12)
    x, eps, xc = rnd(n, 40), rnd(n, 41), rnd(n, 42)
    net = rnd((4, 4, 10, 12), 43)
    x_hat = torch.empty(n, device="cuda")
    net_in = torch.empty((4, 4, 10, 12), device="cuda")
    ops.edm_pre(x.cuda(), eps.cuda(), 0.37, 0.21, x_hat, net_in)
    ref_hat = x + eps * 0.37
    close(x_hat.cpu(), ref_hat, 1e-6, 1e-6)
    close(net_in.cpu(), torch.cat([ref_hat * 0.21] * 2), 1e-6, 1e-6)
    x_next = torch.empty(n, device="cuda")
    ops.edm_post(x_hat, net.cuda(), xc.cuda(), -3.1, 2.5, 0.4, 3.3, -0.9, x_next)
    den = torch.cat([ref_hat] * 2) + net * -3.1
    u, c = den.chunk(2)
    d = u + 2.5 * (c - u)
    d = d - (d - xc) * 0.4
    ref = ref_hat + (ref_hat - d) / 3.3 * -0.9
    close(x_next.cpu(), ref, 1e-5, 1e-5)
    out = torch.empty(n, device="cuda")
    ops.cfg_combine(den.cuda(), torch.tensor([2.5, 1.5], device="cuda"), out)
    close(out.cpu(), u + torch.tensor([2.5, 1.5]).view(2, 1, 1, 1) * (c - u), 1e-6, 1e-6)
    ops.axpby_f32(x.cuda(), 0.3, eps.cuda(), -1.2, out)
    close(out.cpu(), x * 0.3 - eps * 1.2, 1e-6, 1e-6)
    # K12: bit-exact against the reference's sequential accumulation
    N, C, H, W, T = 1, 4, 40, 28, 16
    wins = osamp.sliding_windows(H, W, T, 8)
    tiles = rnd((len(wins), N, C, T, T), 44)
    wts = torch.tensor(osamp.gaussian_weights(T, T))
    x_next, count = torch.zeros(N, C, H, W), torch.zeros(N, C, H, W)
    tw = wts.repeat(N, C, 1, 1)
    for j, (hi, he, wi, we) in enumerate(wins):
        x_next[:, :, hi:he, wi:we] += tiles[j] * tw
        count[:, :, hi:he, wi:we] += tw
    x_next /= count
    out = torch.empty(N, C, H, W, device="cuda")
    ops.tile_blend(tiles.cuda(), torch.tensor(wins, dtype=torch.int32).cuda(), T, wts.cuda(), out)
    assert torch.equal(out.cpu(), x_next), float((out.cpu() - x_next).abs().max())
    mom = rnd((2, 8, 6, 7), 45)
    e = rnd((2, 4, 6, 7), 46)
    z = torch.empty(2, 4, 6, 7, device="cuda")
    from oracle.vae import gaussian_latent
    ops.gaussian_latent(mom.cuda(), e.cuda(), 0.13025, z)
    close(z.cpu(), gaussian_latent(mom, e), 1e-6, 1e-5)
    ops.gaussian_latent(mom.cuda(), None, 0.13025, z)
    close(z.cpu(), gaussian_latent(mom, None), 1e-7, 1e-6)


def test_gemm_conv_attention_vs_torch():
    ops = _ops()
    a = rnd((500, 640), 50).to(BF)
    w = (rnd((1280, 640), 51) * 0.04).to(BF)
    out = torch.empty(500, 1280, dtype=BF, device="cuda")
    ops.gemm(a.cuda(), w.cuda(), out)
    close(out.float().cpu(), a.float() @ w.float().t(), 3e-2)
    B, H, W, Ci, Co = 2, 24, 20, 128, 192
    x = rnd((B, Ci, H, W), 52).to(BF)
    wc = (rnd((Co, Ci, 3, 3), 53) * 0.03).to(BF)
    from supir_b200.nets import pack_conv3x3
    o = torch.empty(B * H * W, Co, dtype=BF, device="cuda")
    ops.conv3x3(nhwc(x.float()), B, H, W, pack_conv3x3(wc).cuda(), o)
    close(from_nhwc(o, B, H, W), F.conv2d(x.float(), wc.float(), padding=1), 3e-2)
    heads, L, Lk = 5, 300, 77
    q, k, v = rnd((B, L, heads * 64), 54).to(BF), rnd((B, Lk, heads * 64), 55).to(BF), rnd((B, Lk, heads * 64), 56).to(BF)
    att = torch.empty(B * L, heads * 64, dtype=BF, device="cuda")
    ops.attention(q.reshape(B * L, -1).cuda(), k.reshape(B * Lk, -1).cuda(), v.reshape(B * Lk, -1).cuda(), att, B, heads, L, Lk)
    qh, kh, vh = (t.float().view(B, -1, heads, 64).transpose(1, 2) for t in (q, k, v))
    ref = F.scaled_dot_product_attention(qh, kh, vh).transpose(1, 2).reshape(B * L, -1)
    close(att.float().cpu(), ref, 2e-2)


def test_colorfix_vs_reference_golden():
    """fp32 image-space ops: 2e-5 against the reference's own outputs."""
    import os
    from supir_b200 import colorfix
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "colorfix.npz"))
    content, style = rnd((1, 3, 70, 90), 900) * 0.5, rnd((1, 3, 70, 90), 901) * 0.5 + 0.1
    hi, lo = colorfix.wavelet_decomposition(content.cuda())
    close(hi.cpu(), torch.from_numpy(g["high"]), 2e-5, 1e-5)
    close(lo.cpu(), torch.from_numpy(g["low"]), 2e-5, 1e-5)
    close(colorfix.wavelet_reconstruction(content.cuda(), style.cuda()).cpu(), torch.from_numpy(g["wavelet"]), 2e-5, 1e-5)
    close(colorfix.adaptive_instance_normalization(content.cuda(), style.cuda()).cpu(), torch.from_numpy(g["adain"]), 2e-5, 1e-5)


def test_tensor2pil_bicubic_uint8_matches_torch():
    """supir_image_to_uint8_bicubic vs the reference's Tensor2PIL arithmetic (SUPIR/util.py:87-94) computed by torch."""
    from supir_b200 import util
    x = (rnd((3, 96, 160), 77) * 0.6).clamp(-1.2, 1.2)
    for h0, w0 in ((96, 160), (75, 131), (200, 333), (48, 80)):
        ref = F.interpolate(x[None], size=(h0, w0), mode="bicubic")
        ref = (ref[0].permute(1, 2, 0) * 127.5 + 127.5).numpy().clip(0, 255).astype(np.uint8)
        got = util.tensor_to_uint8(x.cuda(), h0, w0).cpu().numpy()
        assert got.shape == ref.shape and got.dtype == np.uint8
        diff = np.abs(got.astype(np.int32) - ref.astype(np.int32))
        # the truncation to uint8 turns a last-bit difference of the fp32 interpolation into one grey level now and then
        assert diff.max() <= 1 and (diff != 0).mean() <= 2e-3, (h0, w0, int(diff.max()), float((diff != 0).mean()))
        if (h0, w0) == (96, 160):
            assert diff.max() == 0          # same size: the bicubic kernel is the identity


@pytest.mark.parametrize("M,C,N,with_res", [(3000, 640, 1920, False), (1111, 1280, 1280, True), (129, 320, 96, False)])
def test_gemm_with_folded_layernorm(M, C, N, with_res):
    """Linear(LayerNorm(x)) as statistics pass + GEMM with the normalisation in its epilogue (attention.py:465-486) vs torch fp32."""
    ops = _ops()
    x = (rnd((M, C), 91) * 1.7 + 0.4).to(BF)
    w = rnd((N, C), 92) / C ** 0.5
    g, b = rnd((C,), 93) * 0.2 + 1, rnd((C,), 94) * 0.2
    bias = rnd((N,), 95) * 0.1
    res = rnd((M, N), 96).to(BF) if with_res else None
    ref = F.layer_norm(x.float(), (C,), g, b, 1e-5).to(BF).float() @ w.to(BF).float().t() + bias.to(BF).float()
    if res is not None:
        ref = ref.to(BF).float() + res.float()
    wg, c1, b2 = ops.fold_layernorm(w.cuda(), bias.cuda(), g.cuda(), b.cuda())
    stats = torch.empty(M, 2, dtype=torch.float32, device="cuda")
    ops.layernorm_stats(x.cuda(), stats)
    xf = x.float()
    rstd = (xf.var(1, unbiased=False) + 1e-5).rsqrt()
    close(stats[:, 0].cpu(), rstd, 1e-4, 1e-4)
    close(stats[:, 1].cpu(), xf.mean(1) * rstd, 1e-4, 1e-4)
    out = torch.empty(M, N, dtype=BF, device="cuda")
    ops.gemm(x.cuda(), wg, out, bias=b2, residual=None if res is None else res.cuda(), ln=(stats, c1))
    close(out.float().cpu(), ref, 4e-2, 3e-2)


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 32, 32, 64, 96), (1, 37, 51, 128, 128), (3, 16, 24, 320, 320), (1, 150, 150, 64, 64)])
def test_strided_and_subpixel_convs(B, H, W, Cin, Cout):
    """supir_conv_geom_bf16: 3x3 stride 2 with pad 1 (openaimodel.py:196-210) and with the VAE's (0,1,0,1) padding
    (model.py:81-85) via TMA element strides; nearest-2x + 3x3 (openaimodel.py:131-151) as four sub-pixel 2x2 convolutions."""
    ops = _ops()
    x = rnd((B, Cin, H, W), 101).to(BF)
    w = (rnd((Cout, Cin, 3, 3), 102) / (9 * Cin) ** 0.5).to(BF)
    b = (rnd((Cout,), 103) * 0.1).to(BF).float()
    xt = nhwc(x.float())
    wp = w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous().cuda()
    for pad_lo in (1, 0):
        if pad_lo:
            ref = F.conv2d(x.float(), w.float(), b, stride=2, padding=1)
        else:
            ref = F.conv2d(F.pad(x.float(), (0, 1, 0, 1)), w.float(), b, stride=2, padding=0)
        Ho, Wo = ref.shape[2], ref.shape[3]
        out = torch.full((B * Ho * Wo, Cout), float("nan"), dtype=BF, device="cuda")
        ops.conv3x3_stride2(xt, B, H, W, wp, out, pad_lo, bias=b.cuda())
        close(from_nhwc(out, B, Ho, Wo), ref, 3e-2)
    ref = F.conv2d(F.interpolate(x.float(), scale_factor=2, mode="nearest"), w.float(), b, padding=1)
    out = torch.full((B * 4 * H * W, Cout), float("nan"), dtype=BF, device="cuda")
    ops.upsample2x_conv3x3(xt, B, H, W, [m.cuda() for m in ops.fold_upsample_weights(w.float())], out, bias=b.cuda())
    close(from_nhwc(out, B, 2 * H, 2 * W), ref, 3e-2)
