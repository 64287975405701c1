// supir_b200 — K7/K8/K10/K11/K12/K14 of SURVEY.md §2a and assorted data-movement kernels (HBM-bound, vectorised).
#include "common.cuh"
#include "supir_b200.h"

namespace supir {

static inline unsigned blocks_for(long long n, int threads) {
    long long b = (n + threads - 1) / threads;
    const long long cap = device_sm_count() * 32LL;   // grid-stride loops: 32 blocks per SM
    if (b > cap) b = cap;
    if (b < 1) b = 1;
    return (unsigned)b;
}

// nearest-neighbour 2x upsample on NHWC bf16 (openaimodel.py:131-151, model.py:64-68; value-preserving in any dtype)
__global__ void upsample2x_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, __nv_bfloat16* __restrict__ y,
                                  long long ldy, int B, int H, int W, int C) {
    const int cv = C >> 3;
    const long long total = (long long)B * (2 * H) * (2 * W) * cv;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % cv);
        long long p = i / cv;
        const int xo = (int)(p % (2 * W)); p /= (2 * W);
        const int yo = (int)(p % (2 * H));
        const int b = (int)(p / (2 * H));
        const uint4 u = __ldg(reinterpret_cast<const uint4*>(x + (((long long)b * H + (yo >> 1)) * W + (xo >> 1)) * ldx + c * 8));
        *reinterpret_cast<uint4*>(y + (((long long)b * 2 * H + yo) * 2 * W + xo) * ldy + c * 8) = u;
    }
}

// im2col for the stride-2 3x3 convolutions (UNet Downsample: pad 1 all round, openaimodel.py:196-210;
// VAE Downsample: pad (0,1,0,1), model.py:81-85): out[(b,yo,xo), tap*C + c] = x[b, 2*yo+dy-pad_lo, 2*xo+dx-pad_lo, c]
__global__ void im2col_s2_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, __nv_bfloat16* __restrict__ out,
                                 int B, int H, int W, int C, int Ho, int Wo, int pad_lo) {
    const int cv = C >> 3;
    const long long total = (long long)B * Ho * Wo * 9 * cv;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % cv);
        long long r = i / cv;
        const int tap = (int)(r % 9); r /= 9;
        const int xo = (int)(r % Wo); r /= Wo;
        const int yo = (int)(r % Ho);
        const int b = (int)(r / Ho);
        const int yy = 2 * yo + tap / 3 - pad_lo, xx = 2 * xo + tap % 3 - pad_lo;
        uint4 u = make_uint4(0, 0, 0, 0);
        if (yy >= 0 && yy < H && xx >= 0 && xx < W)
            u = __ldg(reinterpret_cast<const uint4*>(x + (((long long)b * H + yy) * W + xx) * ldx + c * 8));
        *reinterpret_cast<uint4*>(out + (((long long)b * Ho + yo) * Wo + xo) * (9LL * C) + (long long)tap * C + c * 8) = u;
    }
}

__global__ void copy2d_kernel(const __nv_bfloat16* __restrict__ s, long long lds, __nv_bfloat16* __restrict__ d,
                              long long ldd, long long rows, int cols) {
    const int cv = cols >> 3;
    const long long total = rows * cv;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / cv;
        const int c = (int)(i % cv);
        *reinterpret_cast<uint4*>(d + r * ldd + c * 8) = __ldg(reinterpret_cast<const uint4*>(s + r * lds + c * 8));
    }
}

// Row quantization to e4m3 for supir_gemm_fp8 (the attention output before to_out, the GEGLU output before ff.net.2): one warp
// per row, grid-stride over rows; pass 1 takes the row's amax, pass 2 re-reads the row (from L1 / L2) and writes the codes
// (common.cuh e4m3_row_scale / pack_e4m3x4). cols % 8 == 0.
__global__ void quantize_rows_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, uint8_t* __restrict__ q, long long ldq,
                                     float* __restrict__ scale, long long rows, int cols) {
    const int lane = threadIdx.x & 31;
    const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5);
    const int cv = cols >> 3;
    for (long long r = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < rows; r += nwarps) {
        const __nv_bfloat16* xr = x + r * ldx;
        float amax = 0.f;
        for (int c = lane; c < cv; c += 32) {
            const uint4 u = __ldg(reinterpret_cast<const uint4*>(xr + c * 8));
            const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                const float2 f = unpack_bf16x2(w[t]);
                amax = fmaxf(amax, fmaxf(fabsf(f.x), fabsf(f.y)));
            }
        }
        float sc, inv;
        e4m3_row_scale(warp_max(amax), sc, inv);
        if (lane == 0) scale[r] = sc;
        for (int c = lane; c < cv; c += 32) {
            const uint4 u = __ldg(reinterpret_cast<const uint4*>(xr + c * 8));
            const float2 f0 = unpack_bf16x2(u.x), f1 = unpack_bf16x2(u.y), f2 = unpack_bf16x2(u.z), f3 = unpack_bf16x2(u.w);
            const uint32_t lo = pack_e4m3x4(f0.x * inv, f0.y * inv, f1.x * inv, f1.y * inv);
            const uint32_t hi = pack_e4m3x4(f2.x * inv, f2.y * inv, f3.x * inv, f3.y * inv);
            __stcs(reinterpret_cast<uint2*>(q + r * ldq + c * 8), make_uint2(lo, hi));
        }
    }
}

// out = a + y * (*scale)   (ZeroCrossAttn: x_in + x * control_scale, SUPIR_v0.py:150); E: 16-bit storage type (common.cuh)
template <class E>
__global__ void axpy_kernel(const typename E::T* __restrict__ a, long long lda, const typename E::T* __restrict__ y,
                            long long ldy, typename E::T* __restrict__ o, long long ldo, long long rows, int cols,
                            const float* __restrict__ scale) {
    const float s = *scale;
    const int cv = cols >> 3;
    const long long total = rows * cv;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / cv;
        const int c = (int)(i % cv);
        const uint4 ua = __ldg(reinterpret_cast<const uint4*>(a + r * lda + c * 8));
        const uint4 uy = __ldg(reinterpret_cast<const uint4*>(y + r * ldy + c * 8));
        const uint32_t wa[4] = {ua.x, ua.y, ua.z, ua.w}, wy[4] = {uy.x, uy.y, uy.z, uy.w};
        uint32_t w[4];
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const float2 fa = E::unpack2(wa[t]), fy = E::unpack2(wy[t]);
            w[t] = E::pack2(fa.x + E::round(fy.x * s), fa.y + E::round(fy.y * s));
        }
        *reinterpret_cast<uint4*>(o + r * ldo + c * 8) = make_uint4(w[0], w[1], w[2], w[3]);
    }
}

// layout conversions between the reference's NCHW fp32 tensors and the backend's NHWC bf16 activations
__global__ void nchw_f32_to_nhwc_bf16_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y, long long ldy,
                                             int B, int C, int HW) {
    const long long total = (long long)B * C * HW;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const long long r = i / C;  // b*HW + p
        const long long b = r / HW, p = r % HW;
        y[r * ldy + c] = __float2bfloat16_rn(x[(b * C + c) * HW + p]);
    }
}
__global__ void nhwc_bf16_to_nchw_f32_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, float* __restrict__ y,
                                             int B, int C, int HW) {
    const long long total = (long long)B * C * HW;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long p = i % HW;
        const long long bc = i / HW;
        const long long b = bc / C, c = bc % C;
        y[i] = __bfloat162float(x[(b * HW + p) * ldx + c]);
    }
}
// crop window of an NHWC 16-bit tile -> fp32 NCHW view with arbitrary strides (tiled-VAE paste; UNet output)
template <class E>
__global__ void nhwc_crop_to_nchw_f32_kernel(const typename E::T* __restrict__ x, long long ldx, float* __restrict__ y,
                                                  long long ob, long long oc, long long oy, int B, int H, int W, int C,
                                                  int cy0, int cx0, int ch, int cw) {
    const long long total = (long long)B * C * ch * cw;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int xo = (int)(i % cw);
        long long r = i / cw;
        const int yo = (int)(r % ch); r /= ch;
        const int c = (int)(r % C);
        const int b = (int)(r / C);
        y[b * ob + c * oc + yo * oy + xo] = E::to_f(x[(((long long)b * H + yo + cy0) * W + xo + cx0) * ldx + c]);
    }
}
template <class E>
__global__ void f32_to_16_kernel(const float* __restrict__ x, typename E::T* __restrict__ y, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        y[i] = E::from_f(x[i]);
}

// sinusoidal timestep embedding (sgm/modules/diffusionmodules/util.py:206-230): [cos(t f_i) | sin(t f_i)], f_i = exp(-ln(1e4) i / half)
__global__ void timestep_embedding_kernel(const float* __restrict__ t, float* __restrict__ out, int B, int dim) {
    const int half = dim / 2;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * half) return;
    const int b = i / half, k = i % half;
    const float freq = expf(-logf(10000.0f) * (float)k / (float)half);
    const float a = t[b] * freq;
    out[b * dim + k] = cosf(a);
    out[b * dim + half + k] = sinf(a);
}

// y[b, n] = act_out( sum_k act_in(x[b, k]) * W[n, k] + bias[n] )  for tiny batch (M <= 8): one warp per output column.
// Inputs/outputs are rounded to E at the points autocast rounds them (Linear inputs and outputs).
template <int MAXB, class E>
__global__ void linear_small_m_kernel(const float* __restrict__ x, int ldx, const typename E::T* __restrict__ W,
                                      const float* __restrict__ bias, float* __restrict__ y, int ldy, int B, int N,
                                      int K, int silu_in, int silu_out, const float* __restrict__ add, int ldadd) {
    const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (n >= N) return;
    float acc[MAXB];
#pragma unroll
    for (int b = 0; b < MAXB; ++b) acc[b] = 0.f;
    const typename E::T* w = W + (long long)n * K;
    for (int k0 = lane * 8; k0 < K; k0 += 256) {
        const uint4 u = __ldg(reinterpret_cast<const uint4*>(w + k0));
        const uint32_t ww[4] = {u.x, u.y, u.z, u.w};
        float wf[8];
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const float2 f = E::unpack2(ww[t]);
            wf[2 * t] = f.x; wf[2 * t + 1] = f.y;
        }
#pragma unroll
        for (int b = 0; b < MAXB; ++b) {
            if (b < B) {
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    float xv = x[b * ldx + k0 + j];
                    if (silu_in) xv = silu_f(E::round(xv));
                    acc[b] += E::round(xv) * wf[j];
                }
            }
        }
    }
#pragma unroll
    for (int b = 0; b < MAXB; ++b) {
        if (b < B) {
            float v = warp_sum(acc[b]);
            if (lane == 0) {
                v = E::round(v + (bias ? bias[n] : 0.f));
                if (silu_out & 1) v = E::round(silu_f(v));
                if (add) v = E::round(v + add[b * ldadd + n]);
                if (silu_out & 2) v = E::round(silu_f(v));     // SiLU of the sum: what every consumer of `emb` applies first
                y[b * ldy + n] = v;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// EDM sampler elementwise (sgm/modules/diffusionmodules/sampling.py:548-570, denoiser.py:66-73, guiders.py:59-63)
// ---------------------------------------------------------------------------------------------
// x_hat = x + eps * s_noise * sqrt(sigma_hat^2 - sigma^2)  (if gamma > 0);  net_in[0:N] = net_in[N:2N] = x_hat * c_in
__global__ void edm_pre_kernel(const float* __restrict__ x, const float* __restrict__ eps, float noise_mul, float c_in,
                               float* __restrict__ x_hat, float* __restrict__ net_in, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        float v = x[i];
        if (eps) v = v + eps[i] * noise_mul;
        x_hat[i] = v;
        const float s = v * c_in;
        net_in[i] = s;
        net_in[n + i] = s;
    }
}
// denoised_{u,c} = net_{u,c} * c_out + x_hat ; CFG ; restore guidance ; Euler step
__global__ void edm_post_kernel(const float* __restrict__ x_hat, const float* __restrict__ net, const float* __restrict__ x_center,
                                float c_out, float cfg_scale, float restore_mul, float sigma_hat, float dt,
                                float* __restrict__ x_next, float* __restrict__ denoised_out, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float xh = x_hat[i];
        const float du = net[i] * c_out + xh;
        const float dc = net[n + i] * c_out + xh;
        float den = du + cfg_scale * (dc - du);
        if (x_center) {
            const float dcen = den - x_center[i];
            den = den - dcen * restore_mul;
        }
        const float d = (xh - den) / sigma_hat;
        x_next[i] = xh + d * dt;
        if (denoised_out) denoised_out[i] = den;
    }
}


// out = a * alpha + b * beta (fp32; b may be NULL) — the unfused forms of the sampler arithmetic, used when the
// reference's own denoiser/guider objects drive the loop (denoiser.py:73, sampling.py:556, 567-569)
__global__ void axpby_f32_kernel(const float* __restrict__ a, float alpha, const float* __restrict__ b, float beta,
                                 float* __restrict__ out, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        out[i] = a[i] * alpha + (b ? b[i] * beta : 0.f);
}
// LinearCFG / VanillaCFG combine (guiders.py:59-63, sampling_utils.py:7-9): out[n] = u + s_n (c - u), x = [u ; c]
__global__ void cfg_combine_kernel(const float* __restrict__ x, const float* __restrict__ scale, float* __restrict__ out,
                                   int N, long long per) {
    const long long total = (long long)N * per;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const float u = x[i], c = x[total + i];
        out[i] = u + scale[i / per] * (c - u);
    }
}


// K12 gather: out[j, n, c, :, :] = src[n, c, hi_j : hi_j + tile, wi_j : wi_j + tile]  (sampling.py:633-641 slices)
__global__ void tile_gather_kernel(const float* __restrict__ src, const int* __restrict__ win, int num_win, int tile,
                                   float* __restrict__ out, int N, int C, int H, int W) {
    const long long total = (long long)num_win * N * C * tile * tile;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int tx = (int)(i % tile);
        const int ty = (int)((i / tile) % tile);
        const int c = (int)((i / ((long long)tile * tile)) % C);
        const int n = (int)((i / ((long long)tile * tile * C)) % N);
        const int j = (int)(i / ((long long)tile * tile * C * N));
        out[i] = src[(((long long)n * C + c) * H + win[4 * j] + ty) * W + win[4 * j + 2] + tx];
    }
}

// K12: Gaussian-weighted window blend, evaluated per output pixel in the reference's window order so that the fp32
// rounding sequence of `x_next[win] += _x * w; count[win] += w; x_next /= count` (sampling.py:656-659) is reproduced:
// the products and sums are formed in fp64 (w is float64) and rounded to fp32 after every accumulation.
__global__ void tile_blend_kernel(const float* __restrict__ tiles, const int* __restrict__ win, int num_win, int tile,
                                  const double* __restrict__ weights, float* __restrict__ out, int N, int C, int H, int W) {
    const long long total = (long long)N * C * H * W;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % W);
        const int y = (int)((i / W) % H);
        const int c = (int)((i / ((long long)W * H)) % C);
        const int n = (int)(i / ((long long)W * H * C));
        float acc = 0.f, cnt = 0.f;
        for (int j = 0; j < num_win; ++j) {
            const int hi = win[4 * j], he = win[4 * j + 1], wi = win[4 * j + 2], we = win[4 * j + 3];
            if (hi < 0) continue;  // padding slot of a sharded run
            if (y < hi || y >= he || x < wi || x >= we) continue;
            const int ty = y - hi, tx = x - wi;
            const double w = weights[ty * tile + tx];
            const float v = tiles[((((long long)j * N + n) * C + c) * tile + ty) * tile + tx];
            acc = (float)__dadd_rn((double)acc, __dmul_rn((double)v, w));
            cnt = (float)__dadd_rn((double)cnt, w);
        }
        out[i] = acc / cnt;
    }
}

// K14: posterior of the VAE encoder (distributions.py:24-41) fused with the latent scale (SUPIR_model.py:45,61):
// moments [B, 8, hw] fp32 -> z = (mean + exp(0.5 * clamp(logvar, -30, 20)) * eps) * scale   (eps == NULL -> mode())
__global__ void gaussian_latent_kernel(const float* __restrict__ moments, const float* __restrict__ eps, float scale,
                                       float* __restrict__ z, int B, int Cz, long long HW) {
    const long long total = (long long)B * Cz * HW;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long p = i % HW;
        const long long bc = i / HW;
        const long long b = bc / Cz, c = bc % Cz;
        const float mean = moments[(b * 2 * Cz + c) * HW + p];
        float v = mean;
        if (eps) {
            float lv = moments[(b * 2 * Cz + Cz + c) * HW + p];
            lv = fminf(fmaxf(lv, -30.f), 20.f);
            v = mean + expf(0.5f * lv) * eps[i];
        }
        z[i] = scale * v;
    }
}

}  // namespace supir

using namespace supir;
#define ST(s) reinterpret_cast<cudaStream_t>(s)
#define BF(p) reinterpret_cast<__nv_bfloat16*>(p)
#define CBF(p) reinterpret_cast<const __nv_bfloat16*>(p)
#define H16(p) reinterpret_cast<__half*>(p)
#define CH(p) reinterpret_cast<const __half*>(p)
#define DONE()                              \
    do {                                    \
        count_launch();                     \
        SUPIR_CHECK_CUDA(cudaGetLastError()); \
        return SUPIR_OK;                    \
    } while (0)

extern "C" int supir_upsample_nearest2x(const void* x, long long ldx, void* y, long long ldy, int B, int H, int W, int C,
                                        void* stream) {
    SUPIR_REQUIRE(x && y && C % 8 == 0 && ldx % 8 == 0 && ldy % 8 == 0, "supir_upsample_nearest2x: bad args");
    const long long total = (long long)B * 4 * H * W * (C >> 3);
    upsample2x_kernel<<<blocks_for(total, 256), 256, 0, ST(stream)>>>(CBF(x), ldx, BF(y), ldy, B, H, W, C);
    DONE();
}

extern "C" int supir_im2col_3x3_s2(const void* x, long long ldx, void* out, int B, int H, int W, int C, int Ho, int Wo,
                                   int pad_lo, void* stream) {
    SUPIR_REQUIRE(x && out && C % 8 == 0 && ldx % 8 == 0, "supir_im2col_3x3_s2: bad args");
    const long long total = (long long)B * Ho * Wo * 9 * (C >> 3);
    im2col_s2_kernel<<<blocks_for(total, 256), 256, 0, ST(stream)>>>(CBF(x), ldx, BF(out), B, H, W, C, Ho, Wo, pad_lo);
    DONE();
}

extern "C" int supir_copy2d_bf16(const void* src, long long lds, void* dst, long long ldd, long long rows, int cols,
                                 void* stream) {
    SUPIR_REQUIRE(src && dst && cols % 8 == 0 && lds % 8 == 0 && ldd % 8 == 0, "supir_copy2d_bf16: bad args");
    copy2d_kernel<<<blocks_for(rows * (cols >> 3), 256), 256, 0, ST(stream)>>>(CBF(src), lds, BF(dst), ldd, rows, cols);
    DONE();
}

extern "C" int supir_axpy_bf16(const void* a, long long lda, const void* y, long long ldy, void* out, long long ldo,
                               long long rows, int cols, const float* scale, void* stream) {
    SUPIR_REQUIRE(a && y && out && scale && cols % 8 == 0, "supir_axpy_bf16: bad args");
    axpy_kernel<Bf16><<<blocks_for(rows * (cols >> 3), 256), 256, 0, ST(stream)>>>(CBF(a), lda, CBF(y), ldy, BF(out), ldo, rows,
                                                                                   cols, scale);
    DONE();
}

extern "C" int supir_axpy_f16(const void* a, long long lda, const void* y, long long ldy, void* out, long long ldo,
                              long long rows, int cols, const float* scale, void* stream) {
    SUPIR_REQUIRE(a && y && out && scale && cols % 8 == 0, "supir_axpy_f16: bad args");
    axpy_kernel<F16><<<blocks_for(rows * (cols >> 3), 256), 256, 0, ST(stream)>>>(CH(a), lda, CH(y), ldy, H16(out), ldo, rows,
                                                                                  cols, scale);
    DONE();
}

extern "C" int supir_nchw_f32_to_nhwc_bf16(const float* x, void* y, long long ldy, int B, int C, int HW, void* stream) {
    SUPIR_REQUIRE(x && y, "supir_nchw_f32_to_nhwc_bf16: null pointer");
    nchw_f32_to_nhwc_bf16_kernel<<<blocks_for((long long)B * C * HW, 256), 256, 0, ST(stream)>>>(x, BF(y), ldy, B, C, HW);
    DONE();
}

extern "C" int supir_nhwc_bf16_to_nchw_f32(const void* x, long long ldx, float* y, int B, int C, int HW, void* stream) {
    SUPIR_REQUIRE(x && y, "supir_nhwc_bf16_to_nchw_f32: null pointer");
    nhwc_bf16_to_nchw_f32_kernel<<<blocks_for((long long)B * C * HW, 256), 256, 0, ST(stream)>>>(CBF(x), ldx, y, B, C, HW);
    DONE();
}

extern "C" int supir_nhwc_bf16_crop_to_nchw_f32(const void* x, long long ldx, float* y, long long ob, long long oc, long long oy,
                                                int B, int H, int W, int C, int crop_y0, int crop_x0, int crop_h, int crop_w,
                                                void* stream) {
    SUPIR_REQUIRE(x && y, "supir_nhwc_bf16_crop_to_nchw_f32: null pointer");
    SUPIR_REQUIRE(crop_y0 >= 0 && crop_x0 >= 0 && crop_h > 0 && crop_w > 0 && crop_y0 + crop_h <= H && crop_x0 + crop_w <= W,
                  "supir_nhwc_bf16_crop_to_nchw_f32: crop window outside the tile");
    nhwc_crop_to_nchw_f32_kernel<Bf16><<<blocks_for((long long)B * C * crop_h * crop_w, 256), 256, 0, ST(stream)>>>(
        CBF(x), ldx, y, ob, oc, oy, B, H, W, C, crop_y0, crop_x0, crop_h, crop_w);
    DONE();
}

extern "C" int supir_nhwc_f16_crop_to_nchw_f32(const void* x, long long ldx, float* y, long long ob, long long oc, long long oy,
                                               int B, int H, int W, int C, int crop_y0, int crop_x0, int crop_h, int crop_w,
                                               void* stream) {
    SUPIR_REQUIRE(x && y, "supir_nhwc_f16_crop_to_nchw_f32: null pointer");
    SUPIR_REQUIRE(crop_y0 >= 0 && crop_x0 >= 0 && crop_h > 0 && crop_w > 0 && crop_y0 + crop_h <= H && crop_x0 + crop_w <= W,
                  "supir_nhwc_f16_crop_to_nchw_f32: crop window outside the tile");
    nhwc_crop_to_nchw_f32_kernel<F16><<<blocks_for((long long)B * C * crop_h * crop_w, 256), 256, 0, ST(stream)>>>(
        CH(x), ldx, y, ob, oc, oy, B, H, W, C, crop_y0, crop_x0, crop_h, crop_w);
    DONE();
}

extern "C" int supir_quantize_rows(const void* x, long long ldx, void* q, long long ldq, float* scale, long long rows, int cols,
                                   void* stream) {
    SUPIR_REQUIRE(x && q && scale, "supir_quantize_rows: null pointer");
    SUPIR_REQUIRE(rows > 0 && cols > 0 && cols % 8 == 0 && ldx % 8 == 0 && ldq % 8 == 0 && ldx >= cols && ldq >= cols,
                  "supir_quantize_rows: bad shape rows=%lld cols=%d ldx=%lld ldq=%lld (cols, ldx, ldq multiples of 8)", rows, cols, ldx,
                  ldq);
    SUPIR_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(q) & 7) == 0 &&
                  (reinterpret_cast<uintptr_t>(scale) & 3) == 0, "supir_quantize_rows: misaligned pointer (x: 16 bytes, q: 8, scale: 4)");
    quantize_rows_kernel<<<blocks_for(rows * 32, 256), 256, 0, ST(stream)>>>(CBF(x), ldx, reinterpret_cast<uint8_t*>(q), ldq, scale,
                                                                             rows, cols);
    DONE();
}

extern "C" int supir_f32_to_bf16(const float* x, void* y, long long n, void* stream) {
    SUPIR_REQUIRE(x && y && n > 0, "supir_f32_to_bf16: bad args");
    f32_to_16_kernel<Bf16><<<blocks_for(n, 256), 256, 0, ST(stream)>>>(x, BF(y), n);
    DONE();
}

extern "C" int supir_f32_to_f16(const float* x, void* y, long long n, void* stream) {
    SUPIR_REQUIRE(x && y && n > 0, "supir_f32_to_f16: bad args");
    f32_to_16_kernel<F16><<<blocks_for(n, 256), 256, 0, ST(stream)>>>(x, H16(y), n);
    DONE();
}

extern "C" int supir_timestep_embedding(const float* t, float* out, int B, int dim, void* stream) {
    SUPIR_REQUIRE(t && out && dim % 2 == 0, "supir_timestep_embedding: bad args");
    const int n = B * dim / 2;
    timestep_embedding_kernel<<<(n + 127) / 128, 128, 0, ST(stream)>>>(t, out, B, dim);
    DONE();
}

template <class E>
static int linear_small_m_impl(const char* who, const float* x, int ldx, const void* W, const float* bias, float* y, int ldy, int B,
                               int N, int K, int silu_in, int silu_out, const float* add, int ldadd, void* stream) {
    SUPIR_REQUIRE(x && W && y && B >= 1 && B <= 16 && K % 8 == 0, "%s: bad args (B=%d K=%d)", who, B, K);
    const int warps = 8;
    const unsigned blocks = (N + warps - 1) / warps;
    const typename E::T* w = reinterpret_cast<const typename E::T*>(W);
    if (B <= 4)
        linear_small_m_kernel<4, E><<<blocks, warps * 32, 0, ST(stream)>>>(x, ldx, w, bias, y, ldy, B, N, K, silu_in,
                                                                           silu_out, add, ldadd);
    else
        linear_small_m_kernel<16, E><<<blocks, warps * 32, 0, ST(stream)>>>(x, ldx, w, bias, y, ldy, B, N, K, silu_in,
                                                                            silu_out, add, ldadd);
    DONE();
}

extern "C" int supir_linear_small_m(const float* x, int ldx, const void* W, const float* bias, float* y, int ldy, int B,
                                    int N, int K, int silu_in, int silu_out, const float* add, int ldadd, void* stream) {
    return linear_small_m_impl<Bf16>("supir_linear_small_m", x, ldx, W, bias, y, ldy, B, N, K, silu_in, silu_out, add, ldadd, stream);
}

extern "C" int supir_linear_small_m_f16(const float* x, int ldx, const void* W, const float* bias, float* y, int ldy, int B,
                                        int N, int K, int silu_in, int silu_out, const float* add, int ldadd, void* stream) {
    return linear_small_m_impl<F16>("supir_linear_small_m_f16", x, ldx, W, bias, y, ldy, B, N, K, silu_in, silu_out, add, ldadd, stream);
}

extern "C" int supir_edm_pre(const float* x, const float* eps, float noise_mul, float c_in, float* x_hat, float* net_in,
                             long long n, void* stream) {
    SUPIR_REQUIRE(x && x_hat && net_in && n > 0, "supir_edm_pre: bad args");
    edm_pre_kernel<<<blocks_for(n, 256), 256, 0, ST(stream)>>>(x, eps, noise_mul, c_in, x_hat, net_in, n);
    DONE();
}

extern "C" int supir_edm_post(const float* x_hat, const float* net_out, const float* x_center, float c_out,
                              float cfg_scale, float restore_mul, float sigma_hat, float dt, float* x_next,
                              float* denoised, long long n, void* stream) {
    SUPIR_REQUIRE(x_hat && net_out && x_next && n > 0, "supir_edm_post: bad args");
    edm_post_kernel<<<blocks_for(n, 256), 256, 0, ST(stream)>>>(x_hat, net_out, x_center, c_out, cfg_scale, restore_mul,
                                                                sigma_hat, dt, x_next, denoised, n);
    DONE();
}


extern "C" int supir_axpby_f32(const float* a, float alpha, const float* b, float beta, float* out, long long n, void* stream) {
    SUPIR_REQUIRE(a && out && n > 0, "supir_axpby_f32: bad args");
    axpby_f32_kernel<<<blocks_for(n, 256), 256, 0, ST(stream)>>>(a, alpha, b, beta, out, n);
    DONE();
}

extern "C" int supir_cfg_combine(const float* x, const float* scale, float* out, int N, long long per_sample, void* stream) {
    SUPIR_REQUIRE(x && scale && out && N > 0 && per_sample > 0, "supir_cfg_combine: bad args");
    cfg_combine_kernel<<<blocks_for((long long)N * per_sample, 256), 256, 0, ST(stream)>>>(x, scale, out, N, per_sample);
    DONE();
}


extern "C" int supir_tile_gather(const float* src, const int* windows, int num_windows, int tile, float* out, int N, int C,
                                 int H, int W, void* stream) {
    SUPIR_REQUIRE(src && windows && out && num_windows > 0, "supir_tile_gather: bad args");
    tile_gather_kernel<<<blocks_for((long long)num_windows * N * C * tile * tile, 256), 256, 0, ST(stream)>>>(
        src, windows, num_windows, tile, out, N, C, H, W);
    DONE();
}

extern "C" int supir_tile_blend(const float* tiles, const int* windows, int num_windows, int tile, const double* weights,
                                float* out, int N, int C, int H, int W, void* stream) {
    SUPIR_REQUIRE(tiles && windows && weights && out && num_windows > 0, "supir_tile_blend: bad args");
    tile_blend_kernel<<<blocks_for((long long)N * C * H * W, 256), 256, 0, ST(stream)>>>(tiles, windows, num_windows, tile,
                                                                                        weights, out, N, C, H, W);
    DONE();
}

extern "C" int supir_gaussian_latent(const float* moments, const float* eps, float scale, float* z, int B, int Cz,
                                     long long HW, void* stream) {
    SUPIR_REQUIRE(moments && z, "supir_gaussian_latent: null pointer");
    gaussian_latent_kernel<<<blocks_for((long long)B * Cz * HW, 256), 256, 0, ST(stream)>>>(moments, eps, scale, z, B, Cz, HW);
    DONE();
}
